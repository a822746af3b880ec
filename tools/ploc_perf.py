"""TBVH_BUILD_PLOC against the binned builder (tbvh_build, BVH::Build's tree), on the GPU:

  one_tree   the Bistro-sized procedural scene bench.py builds: device time (info.build_ms) and wall time of one build per arm, the arms
             alternated after a warm-up; kernels and host synchronisations of one build of each, counted by torch.profiler in a pass of
             its own (CUB's sort kernels included); SAHCost of both trees; the clustering iterations of the PLOC tree (host restatement,
             tests/ploc_oracle.c, whose tree the device build equals byte for byte)
  batches    tbvh_build_batch over tools/build_batch_perf.py's workloads a (1,000 meshes of 64-20,000 triangles) and b (16 meshes of
             100-500 k and 500 of 100-5,000), flavour PLOC against flavour REFERENCE, alternated
  trace      camera + shadow and one diffuse bounce in the CWBVH layout over both trees of one_tree: Grays/s, alternated, and the hits
             compared (closest t bits and occlusion bits)
  frame      one animation frame with every vertex moved by up to 2 % of the scene's extent: PLOC rebuild + tbvh_convert( CWBVH ) against
             tbvh_refit_layouts of the Build tree (BVH2 and kept CWBVH refitted in place), alternated

  python tools/ploc_perf.py [--reps 5] [--res 1024] [--out DIR]      (needs the GPU; prints one JSON object)
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
sys.path.insert(0, os.path.join(REPO, "tools"))
from tinybvh_b200 import api, _lib, rays as R, scenes  # noqa: E402

ARMS = (("ploc", _lib.BUILD_PLOC), ("build", _lib.BUILD_REFERENCE))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(xs):
    xs = sorted(xs)
    return {"median": xs[len(xs) // 2], "min": xs[0], "max": xs[-1]}


def build(e, v, flavour):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e._build(v, 0, flavour)
    return (time.perf_counter() - t0) * 1e3, e.info().build_ms


def alternate(reps, arms):
    """arms: name -> fn() -> dict of numbers; reps rounds after one warm-up round, the order flipped every round."""
    out = {k: [] for k in arms}
    names = list(arms)
    for k in names:
        arms[k]()
    for r in range(reps):
        for k in (names if r % 2 == 0 else names[::-1]):
            out[k].append(arms[k]())
    return {k: {f: stats([x[f] for x in xs]) for f in xs[0]} for k, xs in out.items()}


def profile_counts(fn):
    """kernels on the device and host synchronisations of one fn() call, from a torch.profiler trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    kernels = syncs = 0
    for ev in p.events():
        name = ev.name
        if ev.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in name.lower() and "memset" not in name.lower():
            kernels += 1
        elif name in ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cudaEventSynchronize", "cudaMemcpy"):
            syncs += 1
    return {"kernels": kernels, "host_syncs": syncs - 1}   # less the synchronise that closes the profiled window


def rate(fn, n, reps=3):
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return n * reps / (a.elapsed_time(b) / 1e3) / 1e9


def one_tree(v, reps):
    from tests import ploc_oracle as po
    es = {k: api.BVH() for k, _ in ARMS}
    arms = {k: (lambda k=k, f=f: dict(zip(("wall_ms", "device_ms"), build(es[k], v, f)))) for k, f in ARMS}
    out = {"times": alternate(reps, arms)}
    for k, f in ARMS:
        out[k] = {"sah": es[k].SAHCost(), "depth": es[k].info().max_depth, "used_nodes": es[k].info().used_nodes,
                  **profile_counts(lambda k=k, f=f: es[k]._build(v, 0, f))}
    nodes, idx, iters, sah = po.build(v)
    ploc_nodes, ploc_idx = es["ploc"].download()
    out["ploc"]["iterations"] = iters
    out["ploc"]["equals_restatement"] = bool(ploc_nodes.tobytes() == nodes.tobytes() and np.array_equal(ploc_idx, idx))
    return out, es


def batches(reps):
    from build_batch_perf import workload
    out = {}
    for name in ("a", "b"):
        meshes = workload(name)
        hs = {k: [api.BVH() for _ in meshes] for k, _ in ARMS}

        def run(k, f):
            import torch
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            api.build_batch(hs[k], meshes, flavour=f)
            return {"wall_ms": (time.perf_counter() - t0) * 1e3, "device_ms": hs[k][0].info().build_ms}
        out[f"workload_{name}"] = {"meshes": len(meshes), "tris": int(sum(m.shape[0] // 3 for m in meshes)),
                                   "times": alternate(reps, {k: (lambda k=k, f=f: run(k, f)) for k, f in ARMS})}
        for k, f in ARMS:
            out[f"workload_{name}"][k] = profile_counts(lambda k=k, f=f: api.build_batch(hs[k], meshes, flavour=f))
        del hs
    return out


def trace(v, es, res, reps):
    import torch
    dev = torch.device("cuda", 0)
    lo, hi = scenes.scene_bounds(v)
    cam = R.primary_rays(*R.bounds_camera(lo, hi, "inside"), res, res, 4)
    ref = cam.copy()
    es["build"].Intersect(ref)
    light = (lo + hi) * 0.5 + np.array([0, (hi - lo)[1] * 0.45, 0], np.float32)
    shadow = R.shadow_rays(ref, light, float((hi - lo).max() * 5e-7))
    diffuse = R.diffuse_rays(ref, v)
    for e in es.values():
        api.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_CWBVH))
        e.layout = api.LAYOUT_CWBVH
    hits = {}
    for k, e in es.items():
        c, d = cam.copy(), diffuse.copy()
        e.Intersect(c), e.Intersect(d)
        hits[k] = (c["t"].view(np.uint32).copy(), d["t"].view(np.uint32).copy(), e.IsOccluded(shadow.copy()))
    out = {"rays_per_kind": int(cam.shape[0]),
           "camera_t_bits_differ": int((hits["ploc"][0] != hits["build"][0]).sum()),
           "diffuse_t_bits_differ": int((hits["ploc"][1] != hits["build"][1]).sum()),
           "shadow_bits_equal": bool(np.array_equal(hits["ploc"][2], hits["build"][2]))}
    to_dev = lambda r: torch.from_numpy(r.view(np.uint8).reshape(-1, 128)[:, :64].copy()).to(dev)  # noqa: E731
    dc, ds, dd = to_dev(cam), to_dev(shadow), to_dev(diffuse)
    wc, wd = torch.empty_like(dc), torch.empty_like(dd)   # closest hits shorten the rays in place: each pass starts from a copy
    bits = torch.zeros((ds.shape[0] + 31) // 32, dtype=torch.int32, device=dev)

    def arm(e):
        return {"camera_shadow_grays": rate(lambda: (wc.copy_(dc), e.Intersect(wc), e.IsOccluded(ds, bits)), dc.shape[0] + ds.shape[0]),
                "diffuse_grays": rate(lambda: (wd.copy_(dd), e.Intersect(wd)), dd.shape[0])}
    out["rates"] = alternate(reps, {k: (lambda e=e: arm(e)) for k, e in es.items()})
    return out


def frame(v, reps):
    import torch
    lo, hi = scenes.scene_bounds(v)
    rng = np.random.default_rng(5)
    moved = np.array(v, np.float32)
    moved[:, :3] += (rng.uniform(-1, 1, (moved.shape[0], 3)) * 0.02 * (hi - lo)).astype(np.float32)
    n = moved.shape[0] // 3
    p = api.BVH()
    r = api.BVH().Build(v)
    api.check(_lib.lib().tbvh_convert(r.h, api.LAYOUT_CWBVH))

    def rebuild():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        p._build(moved, 0, _lib.BUILD_PLOC)
        api.check(_lib.lib().tbvh_convert(p.h, api.LAYOUT_CWBVH))
        return {"wall_ms": (time.perf_counter() - t0) * 1e3, "build_device_ms": p.info().build_ms}

    def refit():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        api.check(_lib.lib().tbvh_refit_layouts(r.h, moved.ctypes.data_as(C.c_void_p), 16, n, api.HOST))
        return {"wall_ms": (time.perf_counter() - t0) * 1e3}
    out = {"times": alternate(reps, {"ploc_rebuild_convert": rebuild, "refit_layouts": refit})}
    out["sah_after"] = {"ploc_rebuild": p.SAHCost(), "refit": r.SAHCost()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("ploc_perf.py needs a GPU")
    out = {"card_power_limit_max_sm_clock": card()}
    v = scenes.procedural_scene(2837209)
    out["one_tree"], es = one_tree(v, args.reps)
    print(json.dumps({"one_tree": out["one_tree"]}), flush=True)
    out["trace"] = trace(v, es, args.res, args.reps)
    print(json.dumps({"trace": out["trace"]}), flush=True)
    del es
    out["frame"] = frame(v, args.reps)
    print(json.dumps({"frame": out["frame"]}), flush=True)
    out["batches"] = batches(args.reps)
    out["card_power_limit_max_sm_clock_after"] = card()
    s = json.dumps(out)
    print(s)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "ploc_perf.json"), "w").write(s + "\n")


if __name__ == "__main__":
    main()
