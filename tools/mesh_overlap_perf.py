"""Cost of intersecting triangle pairs (tbvh_mesh_overlap_pairs / tbvh_mesh_overlap_bits) on the GPU, held to the host restatement
(tests/tritri_oracle.c):

  two meshes  the 512 noise-displaced icospheres of tools/signed_distance_perf.py (2,621,440 triangles, BVH::Build) against a copy shifted
              by 0.3 of a sphere radius along x
  self        the same blobs on a grid of pitch 1.6 instead of 3 (neighbours interpenetrate), merged into one mesh
  soup        scenes.procedural_scene( 2837209 ), the Bistro-sized procedural soup, as a self query
  timing      one warm-up call per arm, then --reps rounds of the (pairs, bits) arms in alternating order: device time by CUDA events on the
              engine's stream around each call, wall time by the host clock around the synchronous call (the bits call synchronised)
  counts      raw against unique pairs, kernel launches of each call, and its host synchronisations (stated from the code)
  baseline    the host restatement's pruned walk over the first --cpu-tris triangles of A, timed on this machine's CPU threads; those
              triangles' device pairs and bit words must equal it bit for bit

  python tools/mesh_overlap_perf.py [--reps 5] [--cpu-tris 32768]      (needs the GPU; prints one JSON object)
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
from tests import tritri_oracle as to  # noqa: E402
from signed_distance_perf import blobs, card  # noqa: E402
from tests.test_signed_distance import icosphere, soup  # noqa: E402


def tight_blobs(seed=7, grid=8, pitch=1.6):
    """blobs() on a grid of the given pitch: spheres of radius about 1 to 1.25 cross their neighbours"""
    rng = np.random.default_rng(seed)
    V, F = icosphere(4)
    out = []
    for i in range(grid ** 3):
        c = np.array([i % grid, (i // grid) % grid, i // grid ** 2], np.float64) * pitch
        k = rng.normal(size=(3, 3)) * 2.5
        ph = rng.uniform(0, 2 * np.pi, 3)
        r = 1.0 + 0.25 * np.sin(V @ k + ph).sum(1) / 3
        out.append(soup(c + V * r[:, None], F))
    return np.concatenate(out)


def run(a, b, reps, cpu_tris, vb, va):
    import torch
    L = _lib.lib()
    n = a.triCount
    s = torch.cuda.Stream()
    cnt = C.c_uint64()
    # the first call sizes the buffer; the raw total comes from the restatement's counting pass over the whole tree below
    _lib.check(L.tbvh_mesh_overlap_pairs(a.h, b.h, None, 0, C.byref(cnt), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    m = cnt.value
    out = torch.empty((max(m, 1), 2), dtype=torch.int32, device="cuda")
    words = torch.empty(max((n + 31) // 32, 1), dtype=torch.int32, device="cuda")

    def pairs():
        _lib.check(L.tbvh_mesh_overlap_pairs(a.h, b.h, C.c_void_p(out.data_ptr()), out.shape[0], C.byref(cnt), _lib.DEVICE, C.c_void_p(s.cuda_stream)))

    def bits():
        _lib.check(L.tbvh_mesh_overlap_bits(a.h, b.h, C.c_void_p(words.data_ptr()), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
        s.synchronize()

    arms = {"pairs": pairs, "bits": bits}
    launches = {}
    for name, f in arms.items():
        k0 = api.launch_count()
        f()
        launches[name] = api.launch_count() - k0
    times = {name: {"device_ms": [], "wall_ms": []} for name in arms}
    for r in range(reps):
        order = list(arms) if r % 2 == 0 else list(arms)[::-1]
        for name in order:
            # events on the caller's stream s: for bits they bracket the kernel; the pairs pipeline runs on the engine stream behind s, so
            # for pairs the span also holds the call's host gaps (its synchronisations and allocations)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            t0 = time.perf_counter()
            arms[name]()
            wall = (time.perf_counter() - t0) * 1e3
            torch.cuda.synchronize()
            e1.record(s)
            torch.cuda.synchronize()
            times[name]["wall_ms"].append(wall)
            times[name]["device_ms"].append(e0.elapsed_time(e1))
    med = {name: {k: float(np.median(v)) for k, v in t.items()} | {"all_wall_ms": [round(x, 3) for x in t["wall_ms"]]} for name, t in times.items()}
    got = out[:m].cpu().numpy().view(np.uint32)
    gbits = words.cpu().numpy().view(np.uint32)
    nodes, idx = b.download()
    k = min(cpu_tris, n)
    t0 = time.perf_counter()
    self = a is b
    want, wbits, keys, _ = to.tree(nodes, idx, vb, va[: 3 * k], self=self)
    cpu_s = time.perf_counter() - t0
    sel = got[got[:, 0] < k]
    agree_pairs = bool(np.array_equal(sel, want))
    agree_bits = bool(np.array_equal(gbits[: k // 32], wbits[: k // 32]))
    return {"triangles_a": int(n), "triangles_b": int(b.triCount), "unique_pairs": int(m), "raw_keys_first_k": int(keys.shape[0]),
            "unique_first_k": int(sel.shape[0]), "launches": launches, "host_syncs": {"pairs": 2, "bits": 0},
            "pairs": med["pairs"], "bits": med["bits"], "cpu_walk_tris": int(k), "cpu_walk_s": round(cpu_s, 3),
            "cpu_threads": os.cpu_count(), "agree_pairs": agree_pairs, "agree_bits": agree_bits}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-tris", type=int, default=32768)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    out = {"card": card()}
    if not args.only or "two" in args.only:
        v = blobs()
        w = v.copy()
        w[:, 0] += np.float32(0.3)
        a, b = api.BVH().Build(v), api.BVH().Build(w)
        out["two_meshes"] = run(a, b, args.reps, args.cpu_tris, w, v)
        print(json.dumps(out), flush=True)
    if not args.only or "self" in args.only:
        v = tight_blobs()
        e = api.BVH().Build(v)
        out["self_blobs"] = run(e, e, args.reps, args.cpu_tris, v, v)
        print(json.dumps(out), flush=True)
    if not args.only or "soup" in args.only:
        v = scenes.procedural_scene(2837209)
        e = api.BVH().Build(v)
        out["self_soup"] = run(e, e, args.reps, args.cpu_tris, v, v)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
