"""Cost of signed distances (tbvh_signed_distance_prepare / tbvh_signed_distance) on the GPU against tbvh_closest_point on the same queries,
held to the host restatement (tests/sdf_oracle.c):

  mesh      512 noise-displaced icospheres of 5,120 triangles (2,621,440 triangles, closed and concave) on an 8 x 8 x 8 grid, BVH::Build
  queries   2^22 "near" (points on random triangles jittered by 2 % of a sphere's radius) and 2^22 "uniform" (uniform in the mesh's box)
            device-resident queries, r_max = inf; seeded
  query     one warm-up call per arm, then --reps rounds of the (kind, call) arms in alternating order, each call timed by CUDA events
  prepare   wall time of the synchronous call (--reps calls, median), and device time from one call under torch.profiler (the span from
            the first kernel's start to the last kernel's end, and the sum of kernel times); the same for a cone whose apex joins 131,072
            triangles (one thread sums that vertex's run) against a sphere of the same triangle count
  check     the signed records of the first --cpu-queries queries of each kind equal the restatement's bit for bit

  python tools/signed_distance_perf.py [--reps 10] [--cpu-queries 32768] [--out DIR]      (needs the GPU; prints one JSON object)
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
from tinybvh_b200 import api, _lib  # noqa: E402
from tests import sdf_oracle as so  # noqa: E402
from tests.test_signed_distance import cone, icosphere, soup  # noqa: E402

N = 1 << 22


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def blobs(seed=7, grid=8):
    """grid^3 icospheres of 5,120 triangles, each vertex moved along its radius by smooth noise (closed, concave, disjoint)"""
    rng = np.random.default_rng(seed)
    V, F = icosphere(4)
    out = []
    for i in range(grid ** 3):
        c = np.array([i % grid, (i // grid) % grid, i // grid ** 2], np.float64) * 3.0
        k = rng.normal(size=(3, 3)) * 2.5
        ph = rng.uniform(0, 2 * np.pi, 3)
        r = 1.0 + 0.25 * np.sin(V @ k + ph).sum(1) / 3
        out.append(soup(c + V * r[:, None], F))
    return np.concatenate(out)


def make_queries(v, seed=2026):
    rng = np.random.default_rng(seed)
    tri = v.reshape(-1, 3, 4)[:, :, :3]
    lo, hi = tri.reshape(-1, 3).min(0).astype(np.float64), tri.reshape(-1, 3).max(0).astype(np.float64)
    k = rng.integers(0, tri.shape[0], N)
    w = rng.dirichlet((1, 1, 1), N)
    near = np.einsum("nk,nkd->nd", w, tri[k].astype(np.float64)) + rng.normal(size=(N, 3)) * 0.02
    uni = lo + rng.random((N, 3)) * (hi - lo)
    out = {}
    for name, p in (("near", near), ("uniform", uni)):
        q = np.empty((N, 4), np.float32)
        q[:, :3], q[:, 3] = p, np.inf
        out[name] = q
    return out


def prepare_times(obj, reps):
    """wall ms of the synchronous prepare (median of reps), then device span / kernel sum of one call under the profiler"""
    import torch
    L = _lib.lib()
    _lib.check(L.tbvh_signed_distance_prepare(obj.h))
    wall = []
    for _ in range(reps):
        t0 = time.perf_counter()
        _lib.check(L.tbvh_signed_distance_prepare(obj.h))
        wall.append((time.perf_counter() - t0) * 1e3)
    wall.sort()
    res = {"wall_ms_median": wall[len(wall) // 2], "wall_ms_min": wall[0], "wall_ms_max": wall[-1]}
    n0 = api.launch_count()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _lib.check(L.tbvh_signed_distance_prepare(obj.h))
        torch.cuda.synchronize()
    res["launches"] = api.launch_count() - n0
    ks = [e for e in prof.events() if e.device_type.name == "CUDA" and e.time_range.end > e.time_range.start]
    if ks:
        res["device_span_ms"] = (max(e.time_range.end for e in ks) - min(e.time_range.start for e in ks)) / 1e3
        res["kernel_sum_ms"] = sum(e.time_range.end - e.time_range.start for e in ks) / 1e3
        top = {}
        for e in ks:
            top[e.name] = top.get(e.name, 0) + (e.time_range.end - e.time_range.start) / 1e3
        res["kernels_ms"] = dict(sorted(top.items(), key=lambda x: -x[1])[:6])
    else:
        res["device_span_ms"] = "not measured"
    return res


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
    v = blobs()
    res["triangles"] = v.shape[0] // 3
    e = api.BVH().Build(v)
    res["tree_depth"] = e.info().max_depth
    res["prepare"] = prepare_times(e, a.reps)
    qs = make_queries(v)
    dq = {k: torch.from_numpy(q).cuda() for k, q in qs.items()}
    rec = torch.empty((N, 4), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def call(kind, fn):
        _lib.check(getattr(L, fn)(e.h, C.c_void_p(dq[kind].data_ptr()), C.c_void_p(rec.data_ptr()), N, _lib.DEVICE, C.c_void_p(s.cuda_stream)))

    def timed(kind, fn):
        torch.cuda.synchronize()
        e0.record(s)
        call(kind, fn)
        e1.record(s)
        e1.synchronize()
        return e0.elapsed_time(e1)

    arms = [(k, fn) for k in qs for fn in ("tbvh_closest_point", "tbvh_signed_distance")]
    for arm in arms:
        timed(*arm)
    ms = {arm: [] for arm in arms}
    for r in range(a.reps):
        for arm in (arms if r % 2 == 0 else arms[::-1]):
            ms[arm].append(timed(*arm))
    gpu = {}
    for (k, fn), xs in ms.items():
        xs = sorted(xs)
        gpu[f"{k}/{fn}"] = {"ms_median": xs[len(xs) // 2], "ms_min": xs[0], "ms_max": xs[-1], "gqueries_per_s": N / (xs[len(xs) // 2] * 1e-3) / 1e9}
    res["gpu"] = gpu
    # the restatement over a subset (its pruned walk, then the sign)
    m = a.cpu_queries
    nodes, idx = e.download()
    t0 = time.perf_counter()
    table = so.prepare(v)
    res["host_prepare_s"] = time.perf_counter() - t0
    agree, inside = {}, {}
    for k, q in qs.items():
        sub = np.ascontiguousarray(q[:m])
        want = so.brute(nodes, idx, v, sub, table=table, walk=True)
        call(k, "tbvh_signed_distance")
        s.synchronize()
        got = rec[:m].cpu().numpy()
        agree[k] = bool(np.array_equal(got.view(np.uint32), want.view(np.uint32)))
        inside[k] = float(np.signbit(got[:, 0]).mean())
    res["device_equals_restatement"] = agree
    res["inside_fraction"] = inside
    # the prepare's long runs: a 131,072-triangle fan at one vertex against a sphere of the same size
    Vc, Fc = cone(fan=131072)
    cn = api.BVH().Build(soup(Vc, Fc))
    Vs, Fs = icosphere(7)
    sp = api.BVH().Build(soup(Vs, Fs[: Fc.shape[0]]))
    res["prepare_fan"] = {"triangles": int(Fc.shape[0]), "apex_valence": 131072, "cone": prepare_times(cn, a.reps),
                          "sphere_same_count": prepare_times(sp, a.reps)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "signed_distance_perf.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
