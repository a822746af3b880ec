"""What k costs in multi-hit rays through a TLAS (tbvh_intersect_all_tlas) on the GPU, against the TLAS closest-hit walk
(tbvh_intersect_device, BLASses in the BVH layout) on the same rays:

  scene     1,000 instances (rotated, non-uniformly scaled, translated; seeded) over four procedural BLASses of 10,000, 30,000, 60,000 and
            100,000 triangles built by BVH::Build: an instanced scene of 50 M instanced triangles
  rays      2^20 device-resident 64-byte rays per kind, tmax = 1e30: "camera" (a 1024 x 1024 pinhole view from outside the instances' world
            box, one sample per pixel) and "random" (origins uniform in that box, directions uniform on the sphere); seeded
  arms      per ray kind: tbvh_intersect_all_tlas at k = 1, 4, 16, 64 and tbvh_intersect_device
  timing    one warm-up call per arm, then --reps rounds with the arms in alternating order, each call timed by CUDA events on one stream;
            medians
  check     the first --check-rays rays of every tbvh_intersect_all_tlas arm against the host restatement's pruned walk
            (tests/allhits_tlas_oracle.c), bit for bit

  python tools/intersect_all_tlas_perf.py [--reps 10] [--check-rays 4096] [--out DIR]      (needs the GPU; prints one JSON object)
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tinybvh_b200 import api, _lib, rays as R, scenes  # noqa: E402
from tests import allhits_tlas_oracle as tao, util  # noqa: E402

N = 1 << 20
KS = (1, 4, 16, 64)
BLAS_TRIS = (10_000, 30_000, 60_000, 100_000)
INSTANCES = 1000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make_rays(lo, hi, seed=2026):
    eye, view = R.bounds_camera(lo, hi, "outside")
    cam = R.gpu_records(R.primary_rays(eye, view, 1024, 1024, 1))
    rng = np.random.default_rng(seed)
    O = (lo + rng.random((N, 3)).astype(np.float32) * (hi - lo)).astype(np.float32)
    rnd = R.gpu_records(R.make_rays(O, rng.normal(size=(N, 3)).astype(np.float32)))
    return {"camera": cam, "random": rnd}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--check-rays", type=int, default=4096)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert api.device_count() > 0, "needs the GPU"
    L = _lib.lib()
    res = {"card": card(), "rays_per_kind": N, "instances": INSTANCES, "blas_triangles": list(BLAS_TRIS)}
    verts = [scenes.procedural_scene(n, 40 + i) for i, n in enumerate(BLAS_TRIS)]
    blas = [api.BVH().Build(v) for v in verts]
    inst = np.zeros(INSTANCES, api.BLAS_INSTANCE)
    inst["transform"] = util.random_transforms(INSTANCES, 11, spread=600.0)
    inst["blasIdx"] = np.arange(INSTANCES) % len(blas)
    inst["mask"] = 0xFFFF
    t = api.TLAS().Build(inst, blas)
    res["tlas_depth"] = t.info().max_depth
    lo, hi = inst["aabbMin"].min(0).astype(np.float32), inst["aabbMax"].max(0).astype(np.float32)
    rs = make_rays(lo, hi)
    dr = {kind: torch.from_numpy(r.view(np.uint8).reshape(N, 64).copy()).cuda() for kind, r in rs.items()}
    work = {kind: torch.empty_like(x) for kind, x in dr.items()}
    hits = torch.empty(N * max(KS) * 4, dtype=torch.float32, device="cuda")
    insts = torch.empty(N * max(KS), dtype=torch.int32, device="cuda")
    counts = torch.empty(N, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def call(kind, k):
        if k == 0:
            # the closest-hit walk writes its hits into the records: it walks a fresh copy (the copy is outside the timed window)
            _lib.check(L.tbvh_intersect_device(t.h, _lib.LAYOUT_BVH, C.c_void_p(work[kind].data_ptr()), 64, None, N, C.c_void_p(s.cuda_stream)))
        else:
            _lib.check(L.tbvh_intersect_all_tlas(t.h, C.c_void_p(dr[kind].data_ptr()), 64, N, k, C.c_void_p(hits.data_ptr()), C.c_void_p(insts.data_ptr()),
                                                 C.c_void_p(counts.data_ptr()), _lib.DEVICE, C.c_void_p(s.cuda_stream)))

    def timed(kind, k):
        with torch.cuda.stream(s):
            work[kind].copy_(dr[kind])
        torch.cuda.synchronize()
        e0.record(s)
        call(kind, k)
        e1.record(s)
        e1.synchronize()
        return e0.elapsed_time(e1)

    arms = [(kind, k) for kind in rs for k in (0,) + KS]
    for arm in arms:
        timed(*arm)
    ms = {arm: [] for arm in arms}
    for r in range(a.reps):
        for arm in (arms if r % 2 == 0 else arms[::-1]):
            ms[arm].append(timed(*arm))
    gpu = {}
    for (kind, k), xs in ms.items():
        xs = sorted(xs)
        med = xs[len(xs) // 2]
        gpu[f"{kind}/{'intersect' if k == 0 else f'k{k}'}"] = {"ms_median": med, "ms_min": xs[0], "ms_max": xs[-1]}
    res["gpu"] = gpu
    # the first rays of every arm held to the host restatement, and the counts at k = 64
    m = a.check_rays
    tn, ti = t.download()
    scene = (tn, ti, inst, [(*b.download(), v) for b, v in zip(blas, verts)])
    agree, mean_count = {}, {}
    for kind, r in rs.items():
        sub = np.ascontiguousarray(r[:m])
        for k in KS:
            wh, wi, wc = tao.walk(*scene, sub, k)
            call(kind, k)
            s.synchronize()
            gh = hits[: m * k * 4].cpu().numpy().reshape(m, k, 4)
            gi = insts[: m * k].cpu().numpy().view(np.uint32).reshape(m, k)
            gc = counts[:m].cpu().numpy().view(np.uint32)
            agree[f"{kind}/k{k}"] = bool(np.array_equal(gh.view(np.uint32), wh.view(np.uint32)) and np.array_equal(gi, wi) and np.array_equal(gc, wc))
        call(kind, 64)
        s.synchronize()
        c = counts.cpu().numpy()
        mean_count[kind] = {"mean": float(c.mean()), "saturated_fraction": float((c > 64).mean())}
    res["device_equals_restatement"] = agree
    res["count_at_k64"] = mean_count
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "intersect_all_tlas_perf.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
