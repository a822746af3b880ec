"""Throughput of the proximity queries (tbvh_closest_point / tbvh_sphere_overlap) on the GPU, against the host restatement's pruned walk
(tests/closest_oracle.c) on the host threads:

  scene     the Bistro-sized procedural scene bench.py falls back to (2,837,209 triangles), as BVH::Build and BuildHQ trees
  queries   2^22 device-resident queries per kind: "near" (points on random triangles jittered by 1 % of the scene's extent, r_max = inf),
            "uniform" (uniform in the scene's box, r_max = inf) and "sphere" (the near points as centres, r = 0.5 % of the extent, one bit
            each); seeded
  timing    one warm-up call per tree and kind, then --reps rounds with the (tree, kind) arms in alternating order, each call timed by CUDA
            events on one stream; queries/s from the median
  cpu       orc_cp_walk (the same rules, OpenMP over queries) over the first --cpu-queries queries of each kind, wall time; the device
            results of those queries must equal it bit for bit

  python tools/closest_point_perf.py [--reps 10] [--cpu-queries 32768] [--out DIR]      (needs the GPU; prints one JSON object)
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tinybvh_b200 import api, _lib, scenes  # noqa: E402
from tests import closest_oracle as co  # noqa: E402

N = 1 << 22


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make_queries(v, seed=2026):
    rng = np.random.default_rng(seed)
    tri = v.reshape(-1, 3, 4)[:, :, :3]
    lo, hi = tri.reshape(-1, 3).min(0).astype(np.float64), tri.reshape(-1, 3).max(0).astype(np.float64)
    ext = float((hi - lo).max())
    k = rng.integers(0, tri.shape[0], N)
    w = rng.dirichlet((1, 1, 1), N)
    near = np.einsum("nk,nkd->nd", w, tri[k].astype(np.float64)) + rng.normal(size=(N, 3)) * 0.01 * ext
    uni = lo + rng.random((N, 3)) * (hi - lo)
    out = {}
    for name, p, r in (("near", near, np.inf), ("uniform", uni, np.inf), ("sphere", near, 0.005 * ext)):
        q = np.empty((N, 4), np.float32)
        q[:, :3], q[:, 3] = p, r
        out[name] = q
    return out, ext


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--cpu-queries", type=int, default=32768)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert api.device_count() > 0, "needs the GPU"
    L = _lib.lib()
    res = {"card": card(), "queries_per_kind": N}
    v = scenes.procedural_scene(2837209)
    trees = {"Build": api.BVH().Build(v), "BuildHQ": api.BVH().BuildHQ(v)}
    res["tree_depth"] = {k: t.info().max_depth for k, t in trees.items()}
    qs, ext = make_queries(v)
    dq = {k: torch.from_numpy(q).cuda() for k, q in qs.items()}
    rec = torch.empty((N, 4), dtype=torch.float32, device="cuda")
    bits = torch.empty(N // 32, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def call(t, kind):
        q = C.c_void_p(dq[kind].data_ptr())
        if kind == "sphere":
            _lib.check(L.tbvh_sphere_overlap(trees[t].h, q, C.c_void_p(bits.data_ptr()), N, _lib.DEVICE, C.c_void_p(s.cuda_stream)))
        else:
            _lib.check(L.tbvh_closest_point(trees[t].h, q, C.c_void_p(rec.data_ptr()), N, _lib.DEVICE, C.c_void_p(s.cuda_stream)))

    def timed(t, kind):
        torch.cuda.synchronize()
        e0.record(s)
        call(t, kind)
        e1.record(s)
        e1.synchronize()
        return e0.elapsed_time(e1)

    arms = [(t, k) for t in trees for k in qs]
    for t, k in arms:
        timed(t, k)
    ms = {arm: [] for arm in arms}
    for r in range(a.reps):
        for arm in (arms if r % 2 == 0 else arms[::-1]):
            ms[arm].append(timed(*arm))
    gpu = {}
    for (t, k), xs in ms.items():
        xs = sorted(xs)
        gpu[f"{t}/{k}"] = {"ms_median": xs[len(xs) // 2], "ms_min": xs[0], "ms_max": xs[-1], "gqueries_per_s": N / (xs[len(xs) // 2] * 1e-3) / 1e9}
    res["gpu"] = gpu
    # host restatement over a subset, and the device results of that subset held to it
    m = a.cpu_queries
    cpu, agree = {}, {}
    for t, obj in trees.items():
        nodes, idx = obj.download()
        for k, q in qs.items():
            sub = np.ascontiguousarray(q[:m])
            t0 = time.perf_counter()
            want = co.walk(nodes, idx, v, sub, any_=k == "sphere")
            dt = time.perf_counter() - t0
            cpu[f"{t}/{k}"] = {"s": dt, "mqueries_per_s": m / dt / 1e6}
            call(t, k)
            s.synchronize()
            got = (bits[: m // 32].cpu().numpy().view(np.uint32) if k == "sphere" else rec[:m].cpu().numpy())
            agree[f"{t}/{k}"] = bool(np.array_equal(got.view(np.uint32), want.view(np.uint32)))
    res["cpu"] = {"threads": os.cpu_count(), "queries": m, "arms": cpu}
    res["device_equals_restatement"] = agree
    hits = {}
    for t in trees:
        call(t, "sphere")
        s.synchronize()
        hits[t] = float(np.unpackbits(bits.cpu().numpy().view(np.uint8)).mean())
    res["sphere_hit_fraction"] = hits
    res["extent"] = ext
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "closest_point_perf.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
