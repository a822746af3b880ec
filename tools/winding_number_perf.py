"""Cost of generalized winding numbers (tbvh_winding_number_prepare / tbvh_winding_number) on the GPU, held to the host restatement
(tests/wn_oracle.c):

  meshes    "blobs": the 512 noise-displaced icospheres of tools/signed_distance_perf.py (2,621,440 triangles, closed), and "soup": the
            Bistro-sized procedural soup (scenes.procedural_scene, 2,837,209 triangles, open and self-intersecting); BVH::Build trees
  queries   2^22 "near" (points on random triangles jittered by 0.02) and 2^22 "uniform" (uniform in the mesh's box) device-resident
            queries per mesh, seeded (signed_distance_perf.make_queries); beta = 2 and 4 over all of them, beta = inf (the exact sum,
            every triangle per query) over the first --exact-queries of each kind
  timing    one warm-up call per arm, then --reps rounds of the arms in alternating order, each call timed by CUDA events; on blobs
            tbvh_signed_distance over the same queries is an arm too, as the cost reference
  prepare   wall time of the synchronous call (--reps calls, median), and device time from one call under torch.profiler
  check     the first --cpu-queries results of each kind at beta 2 and 4, and the first --cpu-exact at beta inf, equal the restatement's

  python tools/winding_number_perf.py [--reps 5] [--cpu-queries 32768] [--out DIR]      (needs the GPU; prints one JSON object)
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
from tests import wn_oracle as wo  # noqa: E402
import signed_distance_perf as sdp  # noqa: E402

N = sdp.N


def prepare_times(obj, reps):
    """wall ms of the synchronous prepare (median of reps), then device span / kernel sum of one call under the profiler"""
    import torch
    L = _lib.lib()
    _lib.check(L.tbvh_winding_number_prepare(obj.h))
    wall = []
    for _ in range(reps):
        t0 = time.perf_counter()
        _lib.check(L.tbvh_winding_number_prepare(obj.h))
        wall.append((time.perf_counter() - t0) * 1e3)
    wall.sort()
    res = {"wall_ms_median": wall[len(wall) // 2], "wall_ms_min": wall[0], "wall_ms_max": wall[-1]}
    n0 = api.launch_count()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _lib.check(L.tbvh_winding_number_prepare(obj.h))
        torch.cuda.synchronize()
    res["launches"] = api.launch_count() - n0
    ks = [e for e in prof.events() if e.device_type.name == "CUDA" and e.time_range.end > e.time_range.start]
    if ks:
        res["device_span_ms"] = (max(e.time_range.end for e in ks) - min(e.time_range.start for e in ks)) / 1e3
        res["kernel_sum_ms"] = sum(e.time_range.end - e.time_range.start for e in ks) / 1e3
    else:
        res["device_span_ms"] = "not measured"
    return res


def workload(name, v, a):
    import torch
    L = _lib.lib()
    res = {"triangles": v.shape[0] // 3}
    e = api.BVH().Build(v)
    res["tree_depth"], res["slots"] = e.info().max_depth, e.info().used_nodes
    res["prepare"] = prepare_times(e, a.reps)
    qs = sdp.make_queries(v)
    dq = {k: torch.from_numpy(q).cuda() for k, q in qs.items()}
    out = torch.empty(N, dtype=torch.float32, device="cuda")
    rec = torch.empty((N, 4), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    closed = name == "blobs"
    if closed:
        _lib.check(L.tbvh_signed_distance_prepare(e.h))

    def call(kind, arm):
        n = N if arm != "inf" else a.exact_queries
        qp = C.c_void_p(dq[kind].data_ptr())
        if arm == "signed_distance":
            _lib.check(L.tbvh_signed_distance(e.h, qp, C.c_void_p(rec.data_ptr()), n, _lib.DEVICE, C.c_void_p(s.cuda_stream)))
        else:
            _lib.check(L.tbvh_winding_number(e.h, qp, C.c_void_p(out.data_ptr()), n, float(arm), _lib.DEVICE, C.c_void_p(s.cuda_stream)))

    def timed(kind, arm):
        torch.cuda.synchronize()
        e0.record(s)
        call(kind, arm)
        e1.record(s)
        e1.synchronize()
        return e0.elapsed_time(e1)

    arms = [(k, b) for k in qs for b in ("2", "4", "inf") + (("signed_distance",) if closed else ())]
    for arm in arms:
        timed(*arm)
    ms = {arm: [] for arm in arms}
    for r in range(a.reps):
        for arm in (arms if r % 2 == 0 else arms[::-1]):
            ms[arm].append(timed(*arm))
    gpu = {}
    for (k, b), xs in ms.items():
        xs = sorted(xs)
        n = N if b != "inf" else a.exact_queries
        key = f"{k}/signed_distance" if b == "signed_distance" else f"{k}/beta={b}"
        gpu[key] = {"queries": n, "ms_median": xs[len(xs) // 2], "ms_min": xs[0], "ms_max": xs[-1], "gqueries_per_s": n / (xs[len(xs) // 2] * 1e-3) / 1e9}
    res["gpu"] = gpu
    # the restatement over a subset
    nodes, idx = e.download()
    t0 = time.perf_counter()
    t = wo.Table(nodes, idx, v)
    res["host_prepare_s"] = time.perf_counter() - t0
    agree, inside = {}, {}
    for k, q in qs.items():
        for b, m in (("2", a.cpu_queries), ("4", a.cpu_queries), ("inf", a.cpu_exact)):
            sub = np.ascontiguousarray(q[:m])
            want = t.query(sub, float(b))
            call(k, b)
            s.synchronize()
            got = out[:m].cpu().numpy()
            agree[f"{k}/beta={b}"] = bool(np.array_equal(got.view(np.uint32), want.view(np.uint32)))
            if b == "2":
                inside[k] = float((got > 0.5).mean())
    res["device_equals_restatement"] = agree
    res["fraction_w_above_half_beta2"] = inside
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-queries", type=int, default=32768)
    ap.add_argument("--cpu-exact", type=int, default=512)
    ap.add_argument("--exact-queries", type=int, default=1 << 14)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert api.device_count() > 0, "needs the GPU"
    res = {"card": sdp.card(), "queries_per_kind": N}
    res["blobs"] = workload("blobs", sdp.blobs(), a)
    res["soup"] = workload("soup", scenes.procedural_scene(2837209, 1), a)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "winding_number_perf.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
