"""Cost of distances between meshes (tbvh_mesh_distance / tbvh_mesh_distance_pairs) on the GPU, held to the host restatement
(tests/meshdist_oracle.c):

  clearance   the 512 noise-displaced icospheres of tools/signed_distance_perf.py (2,621,440 triangles, BVH::Build) against a copy shifted
              along x by the blobs' x extent plus 1 % of a sphere radius, so that the copy just clears them: the nearest query at
              r_max = inf (the separation is d.min()) and the pairs within 1 % of a radius
  thin walls  the same blobs as one mesh, the self nearest query at r_max = inf (the nearest triangle sharing no corner)
  soup        scenes.procedural_scene( 2837209 ), the Bistro-sized procedural soup, the self pairs within --soup-r
  timing      one warm-up call per arm, then --reps rounds of the arms in alternating order: device time by CUDA events on the caller's
              stream around each call, wall time by the host clock around the call (the nearest call synchronised)
  counts      kernel launches of each call, and its host synchronisations (stated from the code)
  baseline    the host restatement's pruned walk over the first --cpu-tris triangles of A, timed on this machine's CPU threads; those
              triangles' device records and pairs must equal it bit for bit

  python tools/mesh_distance_perf.py [--reps 5] [--cpu-tris 32768]      (needs the GPU; prints one JSON object)
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
from tinybvh_b200 import api, _lib, scenes  # noqa: E402
from tests import meshdist_oracle as md  # noqa: E402
from signed_distance_perf import blobs, card  # noqa: E402


def timed(arms, reps):
    import torch
    launches = {}
    for name, (f, s) in arms.items():
        k0 = api.launch_count()
        f()
        launches[name] = api.launch_count() - k0
    times = {name: {"device_ms": [], "wall_ms": []} for name in arms}
    for r in range(reps):
        order = list(arms) if r % 2 == 0 else list(arms)[::-1]
        for name in order:
            f, s = arms[name]
            # events on the caller's stream s: for the nearest call they bracket the kernel; the pairs pipeline runs on the engine
            # stream behind s, so for pairs the span also holds the call's host gaps (its synchronisations and allocations)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            t0 = time.perf_counter()
            f()
            wall = (time.perf_counter() - t0) * 1e3
            torch.cuda.synchronize()
            e1.record(s)
            torch.cuda.synchronize()
            times[name]["wall_ms"].append(wall)
            times[name]["device_ms"].append(e0.elapsed_time(e1))
    med = {name: {k: float(np.median(v)) for k, v in t.items()} | {"all_wall_ms": [round(x, 3) for x in t["wall_ms"]]} for name, t in times.items()}
    return med, launches


def run(a, b, reps, cpu_tris, vb, va, nearest=True, r=None):
    import torch
    L = _lib.lib()
    n = a.triCount
    s = torch.cuda.Stream()
    arms, res = {}, {"triangles_a": int(n), "triangles_b": int(b.triCount)}
    rec = torch.empty((n, 2), dtype=torch.float32, device="cuda")
    cnt = C.c_uint64()
    if nearest:
        def near():
            _lib.check(L.tbvh_mesh_distance(a.h, b.h, C.c_float(np.inf), C.c_void_p(rec.data_ptr()), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
            s.synchronize()
        arms["nearest"] = (near, s)
    if r is not None:
        _lib.check(L.tbvh_mesh_distance_pairs(a.h, b.h, C.c_float(r), None, 0, C.byref(cnt), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
        m = cnt.value
        out = torch.empty((max(m, 1), 2), dtype=torch.int32, device="cuda")

        def pairs():
            _lib.check(L.tbvh_mesh_distance_pairs(a.h, b.h, C.c_float(r), C.c_void_p(out.data_ptr()), out.shape[0], C.byref(cnt), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
        arms["pairs"] = (pairs, s)
    med, launches = timed(arms, reps)
    res |= {"launches": launches, "host_syncs": {"nearest": 0, "pairs": 2}} | med
    nodes, idx = b.download()
    k = min(cpu_tris, n)
    self = a is b
    agree = True
    if nearest:
        got = rec.cpu().numpy()
        d, j = got[:, 0], got[:, 1].view(np.uint32)
        t0 = time.perf_counter()
        wd, wj = md.nearest(nodes, idx, vb, va[: 3 * k], self=self)
        res["cpu_nearest_s"] = round(time.perf_counter() - t0, 3)
        agree &= bool(np.array_equal(d[:k].view(np.uint32), wd.view(np.uint32)) and np.array_equal(j[:k], wj))
        res |= {"min_d": float(d.min()), "median_d": float(np.median(d)), "found": int((j != md.NO_PRIM).sum())}
    if r is not None:
        got = out[: cnt.value].cpu().numpy().view(np.uint32)
        t0 = time.perf_counter()
        want, keys, _ = md.pairs(nodes, idx, vb, va[: 3 * k], r, self=self)
        res["cpu_pairs_s"] = round(time.perf_counter() - t0, 3)
        agree &= bool(np.array_equal(got[got[:, 0] < k], want))
        res |= {"r": r, "unique_pairs": int(cnt.value), "raw_keys_first_k": int(keys.shape[0]), "unique_first_k": int(want.shape[0])}
    res |= {"cpu_walk_tris": int(k), "cpu_threads": os.cpu_count(), "agree": agree}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-tris", type=int, default=32768)
    ap.add_argument("--soup-r", type=float, default=1e-3)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    out = {"card": card()}
    v = blobs()
    if not args.only or "clear" in args.only:
        w = v.copy()
        w[:, 0] += np.float32(float(v[:, 0].max() - v[:, 0].min()) + 0.01)
        a, b = api.BVH().Build(v), api.BVH().Build(w)
        out["clearance"] = run(a, b, args.reps, args.cpu_tris, w, v, r=0.01)
        print(json.dumps(out), flush=True)
    if not args.only or "thin" in args.only:
        e = api.BVH().Build(v)
        out["thin_walls"] = run(e, e, args.reps, args.cpu_tris, v, v)
        print(json.dumps(out), flush=True)
    if not args.only or "soup" in args.only:
        v = scenes.procedural_scene(2837209)
        e = api.BVH().Build(v)
        out["self_soup"] = run(e, e, args.reps, args.cpu_tris, v, v, nearest=False, r=args.soup_r)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
