"""Throughput of the sphere casts (tbvh_sphere_cast / tbvh_sphere_cast_occluded) on the GPU, beside the ray walk and the sphere overlap on
the same inputs:

  scene     the Bistro-sized procedural scene bench.py falls back to (2,837,209 triangles), as BVH::Build and BuildHQ trees
  sweeps    2^22 device-resident sweeps per kind, seeded: "short" (from points on random triangles jittered by 1 % of the extent, unit random
            directions, tmax 5 % of the extent) and "long" (from a sphere of radius one extent around the scene's centre to a uniform point
            in its box, D the displacement, tmax 1), each at r = 0.1 % and 1 % of the extent
  arms      cast (16-byte records), occluded (one bit), ray (tbvh_intersect_device on the 64-byte rays with the same O = c, D and hit.t =
            tmax, restored before each call outside the timed window) and overlap (tbvh_sphere_overlap on the starting spheres)
  timing    one warm-up call per arm, then --reps rounds with the arms in alternating order, each call timed by CUDA events on one stream;
            sweeps/s from the median
  check     the device records and bits of the first --check sweeps of each kind must equal the host restatement's pruned walk
            (tests/sweep_oracle.c) bit for bit

  python tools/sphere_cast_perf.py [--reps 7] [--check 32768] [--out DIR]      (needs the GPU; prints one JSON object)
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
from tests import sweep_oracle as so  # noqa: E402

N = 1 << 22


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make_sweeps(v, seed=2026):
    rng = np.random.default_rng(seed)
    tri = v.reshape(-1, 3, 4)[:, :, :3]
    lo, hi = tri.reshape(-1, 3).min(0).astype(np.float64), tri.reshape(-1, 3).max(0).astype(np.float64)
    ext = float((hi - lo).max())
    k = rng.integers(0, tri.shape[0], N)
    w = rng.dirichlet((1, 1, 1), N)
    near = np.einsum("nk,nkd->nd", w, tri[k].astype(np.float64)) + rng.normal(size=(N, 3)) * 0.01 * ext
    d = rng.normal(size=(N, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    mid = (lo + hi) / 2
    s = rng.normal(size=(N, 3))
    far = mid + s / np.linalg.norm(s, axis=1, keepdims=True) * ext
    to = lo + rng.random((N, 3)) * (hi - lo)
    out = {}
    for rname, r in (("r0.1%", 1e-3 * ext), ("r1%", 1e-2 * ext)):
        out[f"short/{rname}"] = so.queries(near, d, r, 0.05 * ext)
        out[f"long/{rname}"] = so.queries(far, to - far, r, 1.0)
    return out, ext


def ray_records(q):
    """64-byte device rays with O = c, D, rD = safercp( D ) and hit.t = tmax"""
    r = np.zeros(q.shape[0], R.GPU_RAY_DTYPE)
    r["O"], r["D"] = q[:, :3], q[:, 4:7]
    r["rD"] = R.safercp(q[:, 4:7])
    r["t"] = q[:, 7]
    r["mask"] = 0xFFFF
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--check", type=int, default=32768)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert api.device_count() > 0, "needs the GPU"
    L = _lib.lib()
    res = {"card": card(), "sweeps_per_kind": N}
    v = scenes.procedural_scene(2837209)
    trees = {"Build": api.BVH().Build(v), "BuildHQ": api.BVH().BuildHQ(v)}
    res["tree_depth"] = {k: t.info().max_depth for k, t in trees.items()}
    qs, ext = make_sweeps(v)
    res["extent"] = ext
    s = torch.cuda.Stream()
    rec = torch.empty((N, 4), dtype=torch.float32, device="cuda")
    bits = torch.empty(N // 32, dtype=torch.int32, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    gpu, agree, hit = {}, {}, {}
    for kind, q in qs.items():
        dq = torch.from_numpy(q).cuda()
        spheres = torch.from_numpy(np.ascontiguousarray(q[:, :4])).cuda()
        rays0 = torch.from_numpy(ray_records(q).view(np.uint8).reshape(N, 64)).cuda()
        rays = torch.empty_like(rays0)

        def call(t, arm):
            h, st = trees[t].h, C.c_void_p(s.cuda_stream)
            if arm == "cast":
                _lib.check(L.tbvh_sphere_cast(h, C.c_void_p(dq.data_ptr()), C.c_void_p(rec.data_ptr()), N, _lib.DEVICE, st))
            elif arm == "occluded":
                _lib.check(L.tbvh_sphere_cast_occluded(h, C.c_void_p(dq.data_ptr()), C.c_void_p(bits.data_ptr()), N, _lib.DEVICE, st))
            elif arm == "ray":
                _lib.check(L.tbvh_intersect_device(h, _lib.LAYOUT_BVH, C.c_void_p(rays.data_ptr()), 64, None, N, st))
            else:
                _lib.check(L.tbvh_sphere_overlap(h, C.c_void_p(spheres.data_ptr()), C.c_void_p(bits.data_ptr()), N, _lib.DEVICE, st))

        def timed(t, arm):
            if arm == "ray":
                with torch.cuda.stream(s):
                    rays.copy_(rays0)
            torch.cuda.synchronize()
            e0.record(s)
            call(t, arm)
            e1.record(s)
            e1.synchronize()
            return e0.elapsed_time(e1)

        arms = [(t, x) for t in trees for x in ("cast", "occluded", "ray", "overlap")]
        for arm in arms:
            timed(*arm)
        ms = {arm: [] for arm in arms}
        for r in range(a.reps):
            for arm in (arms if r % 2 == 0 else arms[::-1]):
                ms[arm].append(timed(*arm))
        for (t, x), xs in ms.items():
            xs = sorted(xs)
            gpu[f"{t}/{kind}/{x}"] = {"ms_median": xs[len(xs) // 2], "ms_min": xs[0], "ms_max": xs[-1],
                                      "gsweeps_per_s": N / (xs[len(xs) // 2] * 1e-3) / 1e9}
        m = a.check
        sub = np.ascontiguousarray(q[:m])
        for t, obj in trees.items():
            nodes, idx = obj.download()
            want = so.walk(nodes, idx, v, sub)
            wbits = so.walk(nodes, idx, v, sub, any_=True)
            call(t, "cast")
            call(t, "occluded")
            s.synchronize()
            got = rec[:m].cpu().numpy()
            gb = bits[: m // 32].cpu().numpy().view(np.uint32)
            agree[f"{t}/{kind}"] = bool(np.array_equal(got.view(np.uint32), want.view(np.uint32)) and np.array_equal(gb, wbits[: m // 32]))
            hit[f"{t}/{kind}"] = float(np.unpackbits(bits.cpu().numpy().view(np.uint8)).mean())
        del dq, spheres, rays0, rays
    res["gpu"] = gpu
    res["device_equals_restatement"] = agree
    res["contact_fraction"] = hit
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "sphere_cast_perf.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
