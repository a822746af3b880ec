"""Animation frame cost of a CWBVH BLAS, BVH::Build tree: tbvh_refit + tbvh_convert against tbvh_refit_layouts (wall and device time, two
alternating rounds), the memory the kept collapse and the refit scratch hold, and the CWBVH traversal rate after the refit against a
fresh conversion of the same moved vertices (what keeping the conversion's collapse costs in tree quality).

  python tools/refit_perf.py [--tris 2837209] [--out DIR]      (needs the GPU; prints one JSON object)
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tinybvh_b200 import api, _lib, rays as R, scenes  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def moved(v, seed, amp):
    rng = np.random.default_rng(seed)
    w = v.copy()
    ext = float((v[:, :3].max(0) - v[:, :3].min(0)).max())
    w[:, :3] += (rng.random((v.shape[0], 3), np.float32) - 0.5) * np.float32(amp * ext)
    return w


def device_span_ms(fn):
    """kernel time and first-kernel-start .. last-kernel-end of one call, from torch.profiler's CUDA activity"""
    import torch
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in p.events() if e.device_type.name == "CUDA" and e.time_range.end > e.time_range.start]
    ker = [e for e in ev if "memcpy" not in e.name.lower() and "memset" not in e.name.lower()]
    if not ev:
        return None
    return {"kernels_ms": sum(e.time_range.elapsed_us() for e in ker) / 1e3, "launches": len(ker),
            "span_ms": (max(e.time_range.end for e in ev) - min(e.time_range.start for e in ev)) / 1e3}


def trace_rate(e, d_rays, reps=5):
    import torch
    e.Intersect(d_rays)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        e.Intersect(d_rays)
    b.record()
    torch.cuda.synchronize()
    return d_rays.shape[0] * reps / (a.elapsed_time(b) / 1e3) / 1e9


def split_total(nodes):
    c = nodes["triCount"].astype(np.int64)
    c[1] = 0
    return nodes.shape[0] + int((2 * (np.maximum((c + 2) // 3, 1) - 1) * (c > 3)).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=2837209)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    v = scenes.procedural_scene(args.tris)
    w = torch.from_numpy(moved(v, 11, 0.02)).to(dev)
    L = _lib.lib()
    out = {"card": card(), "tris": args.tris, "tree": "BVH::Build", "vertices": "device-resident"}

    a = api.BVH8_CWBVH()   # refit + full conversion every frame
    a.build_flavour = _lib.BUILD_REFERENCE
    a.Build(v)
    b = api.BVH8_CWBVH()   # refit over the kept collapse
    b.build_flavour = _lib.BUILD_REFERENCE
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    b.Build(v)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]

    def old():
        api.BVH.Refit(a, w)
        api.check(L.tbvh_convert(a.h, api.LAYOUT_CWBVH))

    def new():
        b.Refit(w)

    new()
    torch.cuda.synchronize()
    free2 = torch.cuda.mem_get_info()[0]
    old()
    rounds = []
    for r in range(2):      # alternating; each timing is a repeat call (first calls above)
        row = {}
        for name, fn in (("refit+convert", old), ("refit_layouts", new)):
            t0 = time.perf_counter()
            fn()
            row[name + "_wall_ms"] = (time.perf_counter() - t0) * 1e3
        row["refit_layouts_build_ms"] = b.info().build_ms
        rounds.append(row)
    out["rounds"] = rounds
    out["device"] = {"refit+convert": device_span_ms(old), "refit_layouts": device_span_ms(new)}
    ia = b.info()
    nodes, _ = api.BVH.download(b)
    out["counts"] = {"bvh2_nodes": ia.used_nodes, "split_nodes": split_total(nodes), "wide_nodes": ia.used_blocks // 5}
    out["memory_mem_get_info_bytes"] = {"build_and_convert": free0 - free1, "first_refit_scratch": free1 - free2}
    # tree quality: the same moved vertices, walked through the kept collapse (b) and through a fresh conversion (a)
    lo, hi = scenes.scene_bounds(moved(v, 11, 0.02))
    rays = R.primary_rays(*R.bounds_camera(lo, hi, "inside"), 1024, 1024, 4)
    d = torch.from_numpy(rays.view(np.uint8).reshape(-1, 128)[:, :64].copy()).to(dev)
    rates = []
    for _ in range(2):
        rates.append({"fresh_conversion_grays": trace_rate(a, d), "kept_collapse_grays": trace_rate(b, d)})
    out["trace_primary_4M"] = rates
    ha, hb = rays.copy(), rays.copy()
    a.Intersect(ha), b.Intersect(hb)
    out["hits_agree"] = float(((ha["prim"] == hb["prim"]) & (ha["t"] == hb["t"])).mean())
    s = json.dumps(out)
    print(s)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "refit_perf.json"), "w").write(s + "\n")


if __name__ == "__main__":
    main()
