"""What k costs in the multi-hit ray query (tbvh_intersect_all) on the GPU, against the closest-hit walk (tbvh_intersect_device, BVH layout)
on the same rays:

  scene     the Bistro-sized procedural scene bench.py falls back to (2,837,209 triangles), as BVH::Build and BuildHQ trees
  rays      2^22 device-resident 64-byte rays per kind, tmax = 1e30: "camera" (a 2048 x 2048 pinhole view from outside the scene's box,
            one sample per pixel) and "random" (origins uniform in the box, directions uniform on the sphere); seeded
  arms      per tree and ray kind: tbvh_intersect_all at k = 1, 2, 4, 16, 64 and tbvh_intersect_device
  timing    one warm-up call per arm, then --reps rounds with the arms in alternating order, each call timed by CUDA events on one
            stream; medians
  check     the first --check-rays rays of every tbvh_intersect_all arm against the host restatement's pruned walk (tests/allhits_oracle.c),
            bit for bit

  python tools/intersect_all_perf.py [--reps 10] [--check-rays 32768] [--out DIR]      (needs the GPU; prints one JSON object)
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
from tests import allhits_oracle as ao  # noqa: E402

N = 1 << 22
KS = (1, 2, 4, 16, 64)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make_rays(v, seed=2026):
    lo, hi = scenes.scene_bounds(v)
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    eye, view = R.bounds_camera(lo, hi, "outside")
    cam = R.gpu_records(R.primary_rays(eye, view, 2048, 2048, 1))
    rng = np.random.default_rng(seed)
    O = (lo + rng.random((N, 3)).astype(np.float32) * (hi - lo)).astype(np.float32)
    rnd = R.gpu_records(R.make_rays(O, rng.normal(size=(N, 3)).astype(np.float32)))
    return {"camera": cam, "random": rnd}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--check-rays", type=int, default=32768)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert api.device_count() > 0, "needs the GPU"
    L = _lib.lib()
    res = {"card": card(), "rays_per_kind": N}
    v = scenes.procedural_scene(2837209)
    trees = {"Build": api.BVH().Build(v), "BuildHQ": api.BVH().BuildHQ(v)}
    res["tree_depth"] = {t: o.info().max_depth for t, o in trees.items()}
    rs = make_rays(v)
    dr = {kind: torch.from_numpy(r.view(np.uint8).reshape(N, 64).copy()).cuda() for kind, r in rs.items()}
    hits = torch.empty(N * max(KS) * 4, dtype=torch.float32, device="cuda")
    counts = torch.empty(N, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def call(t, kind, k):
        rp = C.c_void_p(dr[kind].data_ptr())
        if k == 0:
            _lib.check(L.tbvh_intersect_device(trees[t].h, _lib.LAYOUT_BVH, rp, 64, C.c_void_p(hits.data_ptr()), N, C.c_void_p(s.cuda_stream)))
        else:
            _lib.check(L.tbvh_intersect_all(trees[t].h, rp, 64, N, k, C.c_void_p(hits.data_ptr()), C.c_void_p(counts.data_ptr()), _lib.DEVICE,
                                            C.c_void_p(s.cuda_stream)))

    def timed(*arm):
        torch.cuda.synchronize()
        e0.record(s)
        call(*arm)
        e1.record(s)
        e1.synchronize()
        return e0.elapsed_time(e1)

    arms = [(t, kind, k) for t in trees for kind in rs for k in (0,) + KS]
    for arm in arms:
        timed(*arm)
    ms = {arm: [] for arm in arms}
    for r in range(a.reps):
        for arm in (arms if r % 2 == 0 else arms[::-1]):
            ms[arm].append(timed(*arm))
    gpu = {}
    for (t, kind, k), xs in ms.items():
        xs = sorted(xs)
        med = xs[len(xs) // 2]
        gpu[f"{t}/{kind}/{'intersect' if k == 0 else f'k{k}'}"] = {"ms_median": med, "ms_min": xs[0], "ms_max": xs[-1], "grays_per_s": N / (med * 1e-3) / 1e9}
    res["gpu"] = gpu
    # the first rays of every arm held to the host restatement, and the distribution of counts at k = 64
    m = a.check_rays
    agree, mean_count = {}, {}
    for t, obj in trees.items():
        nodes, idx = obj.download()
        for kind, r in rs.items():
            sub = np.ascontiguousarray(r[:m])
            for k in KS:
                wh, wc = ao.walk(nodes, idx, v, sub, k)
                call(t, kind, k)
                s.synchronize()
                gh = hits[: m * k * 4].cpu().numpy().reshape(m, k, 4)
                gc = counts[:m].cpu().numpy().view(np.uint32)
                agree[f"{t}/{kind}/k{k}"] = bool(np.array_equal(gh.view(np.uint32), wh.view(np.uint32)) and np.array_equal(gc, wc))
            call(t, kind, 64)
            s.synchronize()
            c = counts.cpu().numpy()
            mean_count[f"{t}/{kind}"] = {"mean": float(c.mean()), "saturated_fraction": float((c > 64).mean())}
    res["device_equals_restatement"] = agree
    res["count_at_k64"] = mean_count
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "intersect_all_perf.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
