"""Cost of times of impact between moving meshes (tbvh_mesh_toi / tbvh_mesh_toi_pairs) on the GPU, held to the host restatement
(tests/toi_oracle.c), against the discrete broad phase a caller would otherwise run (tbvh_mesh_distance_pairs at r = eta + xi + twice the
largest displacement of the step, as both triangles of a pair move):

  blobs   the 512 noise-displaced icospheres of tools/signed_distance_perf.py (2,621,440 triangles, BVH::Build) against a copy shifted
          along x by their x extent less 10 % of a sphere radius; within the step A moves 4 % of a radius towards the copy and every
          vertex of both jitters by 0.5 % of a radius
  soup    scenes.procedural_scene( 2837209 ), the Bistro-sized procedural soup, as a self query under a random jitter step
  timing  one warm-up call per arm, then --reps rounds of the arms in alternating order: device time by CUDA events on the caller's
          stream around each call (the pairs calls synchronise the host inside), wall time by the host clock
  check   the restatement over the first --cpu-tris triangles of A, timed on --cpu-threads host threads; those triangles' device records,
          pairs and times must equal it bit for bit.  The iteration histogram counts the nearest records' iters.

  python tools/mesh_toi_perf.py [--reps 5] [--cpu-tris 32768] [--cpu-threads 8]      (needs the GPU; prints one JSON object)
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


def jittered(v, seed, s):
    """every distinct position moved by one normal offset of deviation s: corners a mesh shares stay shared in the end frame, so the self
    query keeps skipping neighbours (corners count as shared when equal in both frames)"""
    rng = np.random.default_rng(seed)
    u, inv = np.unique(v[:, :3], axis=0, return_inverse=True)
    out = v.copy()
    out[:, :3] += (rng.normal(size=(u.shape[0], 3)) * s).astype(np.float32)[inv.reshape(-1)]
    return out


def run(a, a0, a1, b, b0, b1, eta, xi, iters, reps, cpu_tris):
    import torch
    from tinybvh_b200 import _lib
    from tests import toi_oracle as toi
    from mesh_distance_perf import timed
    L = _lib.lib()
    n = a.triCount
    self = a is b
    s = torch.cuda.Stream()
    da0, da1 = torch.from_numpy(a1).cuda(), None
    pa = C.c_void_p(da0.data_ptr())
    if self:
        pb = pa
    else:
        da1 = torch.from_numpy(b1).cuda()
        pb = C.c_void_p(da1.data_ptr())
    disp = max(float(np.abs(a1[:, :3] - a0[:, :3]).max()), float(np.abs(b1[:, :3] - b0[:, :3]).max())) * 3 ** 0.5
    r = float(np.float32(eta) + np.float32(xi) + np.float32(2 * disp))   # both triangles of a pair may close in by disp
    rec = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    cnt, dcnt = C.c_uint64(), C.c_uint64()
    args = (a.h, pa, 16, b.h, pb, 16, C.c_float(eta), C.c_float(xi), iters)
    _lib.check(L.tbvh_mesh_toi_pairs(*args, None, None, 0, C.byref(cnt), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    out = torch.empty((max(cnt.value, 1), 2), dtype=torch.int32, device="cuda")
    tms = torch.empty(max(cnt.value, 1), dtype=torch.float32, device="cuda")
    _lib.check(L.tbvh_mesh_distance_pairs(a.h, b.h, C.c_float(r), None, 0, C.byref(dcnt), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    dout = torch.empty((max(dcnt.value, 1), 2), dtype=torch.int32, device="cuda")

    def near():
        _lib.check(L.tbvh_mesh_toi(*args, C.c_void_p(rec.data_ptr()), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
        s.synchronize()

    def pairs():
        _lib.check(L.tbvh_mesh_toi_pairs(*args, C.c_void_p(out.data_ptr()), C.c_void_p(tms.data_ptr()), out.shape[0], C.byref(cnt), _lib.DEVICE, C.c_void_p(s.cuda_stream)))

    def dpairs():
        _lib.check(L.tbvh_mesh_distance_pairs(a.h, b.h, C.c_float(r), C.c_void_p(dout.data_ptr()), dout.shape[0], C.byref(dcnt), _lib.DEVICE, C.c_void_p(s.cuda_stream)))

    med, launches = timed({"toi_nearest": (near, s), "toi_pairs": (pairs, s), "distance_pairs": (dpairs, s)}, reps)
    res = {"triangles_a": int(n), "triangles_b": int(b.triCount), "eta": eta, "xi": xi, "max_iters": iters, "max_displacement": disp,
           "distance_pairs_r": r, "launches": launches} | med
    got = rec.cpu().numpy()
    t, j, it = got[:, 0], got[:, 2].view(np.uint32), got[:, 3].view(np.uint32)
    found = j != toi.NO_PRIM
    res |= {"contacts": int(found.sum()), "at_t0": int((t[found] == 0).sum()), "unresolved": int((it[found] == iters).sum()),
            "iters_histogram": {int(k): int(c) for k, c in enumerate(np.bincount(it[found], minlength=1)) if c},
            "toi_pair_count": int(cnt.value), "distance_pair_count": int(dcnt.value)}
    nodes, idx = b.download()
    k = min(cpu_tris, n)
    t0 = time.perf_counter()
    want = toi.nearest(nodes, idx, b0, b1, a0[: 3 * k], a1[: 3 * k], eta, xi, iters, self=self)
    res["cpu_nearest_s"] = round(time.perf_counter() - t0, 3)
    t0 = time.perf_counter()
    wp, wt = toi.pairs(nodes, idx, b0, b1, a0[: 3 * k], a1[: 3 * k], eta, xi, iters, self=self)
    res["cpu_pairs_s"] = round(time.perf_counter() - t0, 3)
    gp = out[: cnt.value].cpu().numpy().view(np.uint32)
    gt = tms[: cnt.value].cpu().numpy()
    first = gp[:, 0] < k
    agree = all(np.array_equal(got[:k, c].view(np.uint32), w.view(np.uint32)) for c, w in enumerate(want))
    agree &= bool(np.array_equal(gp[first], wp) and np.array_equal(gt[first].view(np.uint32), wt.view(np.uint32)))
    res |= {"cpu_check_tris": int(k), "cpu_check_pairs": int(wp.shape[0]), "agree": bool(agree)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-tris", type=int, default=32768)
    ap.add_argument("--cpu-threads", type=int, default=8)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    os.environ["OMP_NUM_THREADS"] = str(args.cpu_threads)   # read when the restatement's OpenMP runtime starts
    from tinybvh_b200 import api, scenes
    from signed_distance_perf import blobs, card
    out = {"card": card(), "cpu_threads": args.cpu_threads}
    if not args.only or "blobs" in args.only:
        v = blobs()
        w = v.copy()
        w[:, 0] += np.float32(float(v[:, 0].max() - v[:, 0].min()) - 0.1)
        v1 = jittered(v, 1, 0.005)
        v1[:, 0] += np.float32(0.04)
        w1 = jittered(w, 2, 0.005)
        a, b = api.BVH().Build(v), api.BVH().Build(w)
        out["blobs"] = run(a, v, v1, b, w, w1, 0.002, 0.001, 64, args.reps, args.cpu_tris)
        print(json.dumps(out), flush=True)
    if not args.only or "soup" in args.only:
        v = scenes.procedural_scene(2837209)
        v1 = jittered(v, 3, 5e-4)
        e = api.BVH().Build(v)
        out["self_soup"] = run(e, v, v1, e, v, v1, 0.0, 2.5e-4, 64, args.reps, args.cpu_tris)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
