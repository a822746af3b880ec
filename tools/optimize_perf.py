"""tbvh_optimize on the Bistro-sized procedural scene bench.py builds and on a seeded 150 k-triangle scene, for the Build, BuildAVX and
BuildHQ trees: SAHCost, device and wall time and launches of one call with --rounds rounds, and a trajectory of one-round calls; then camera + shadow rays in the CWBVH
and BVH layouts and one diffuse bounce, before against after, the arms alternated and repeated, with the hits checked.  Each traced pass includes a
device copy of its rays (closest hits shorten them in place), the same in both arms.

The trajectory ("per_round_calls") is a sequence of separate optimize( 1 ) calls.  Each call writes back a renumbered tree, and the
node numbers break ties between equal gains, so these rounds are close to, but not the same as, the rounds of the single call.

  python tools/optimize_perf.py [--rounds 8] [--res 1024] [--out DIR]      (needs the GPU; prints one JSON object)
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


def build(v, flavour, cls=api.BVH):
    e = cls()
    e._build(v, 0, flavour)
    return e


def rate(fn, n, reps):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    out = {"card": card(), "max_rounds": args.rounds, "rays_per_kind": args.res * args.res * 4, "scenes": {}}
    for label, v in (("bistro_sized", scenes.procedural_scene(2837209)), ("seeded_150k", scenes.procedural_scene(150000, 7))):
        lo, hi = scenes.scene_bounds(v)
        cam = R.primary_rays(*R.bounds_camera(lo, hi, "inside"), args.res, args.res, 4)
        rows = {}
        for name, fl in (("Build", _lib.BUILD_REFERENCE), ("BuildAVX", _lib.BUILD_AVX), ("BuildHQ", _lib.BUILD_HQ)):
            row = {}
            before = build(v, fl)
            row["sah_before"] = before.SAHCost()
            # one round per call (not the rounds of the single call below: each call renumbers the tree, and N breaks ties)
            step = build(v, fl)
            per = []
            for _ in range(args.rounds):
                t0 = time.perf_counter()
                r, s = step.optimize(1)
                wall = (time.perf_counter() - t0) * 1e3
                if r == 0:
                    break
                per.append({"sah": s, "device_ms": step.info().build_ms, "wall_ms": wall})
            row["per_round_calls"] = per
            # the whole call
            after = build(v, fl)
            torch.cuda.synchronize()
            n0 = api.launch_count()
            t0 = time.perf_counter()
            r, s = after.optimize(args.rounds)
            row["call"] = {"rounds": r, "sah": s, "device_ms": after.info().build_ms, "wall_ms": (time.perf_counter() - t0) * 1e3,
                           "launches": api.launch_count() - n0, "depth_before": before.info().max_depth, "depth_after": after.info().max_depth}
            # rays: camera, then shadow and diffuse rays from the camera hits of the tree before optimisation
            hb, ha = cam.copy(), cam.copy()
            before.Intersect(hb), after.Intersect(ha)
            row["camera_t_bits_equal"] = bool(np.array_equal(hb["t"].view(np.uint32), ha["t"].view(np.uint32)))
            light = (lo + hi) * 0.5 + np.array([0, (hi - lo)[1] * 0.45, 0], np.float32)
            shadow = R.shadow_rays(hb, light, float((hi - lo).max() * 5e-7))
            diffuse = R.diffuse_rays(hb, v)
            row["shadow_bits_equal"] = bool(np.array_equal(before.IsOccluded(shadow.copy()), after.IsOccluded(shadow.copy())))
            db, da = diffuse.copy(), diffuse.copy()
            before.Intersect(db), after.Intersect(da)
            row["diffuse_t_bits_equal"] = bool(np.array_equal(db["t"].view(np.uint32), da["t"].view(np.uint32)))
            to_dev = lambda r: torch.from_numpy(r.view(np.uint8).reshape(-1, 128)[:, :64].copy()).to(dev)  # noqa: E731
            dc, ds, dd = to_dev(cam), to_dev(shadow), to_dev(diffuse)
            wc, wd = torch.empty_like(dc), torch.empty_like(dd)   # closest hits shorten the rays in place: each pass starts from a copy
            bits = torch.zeros((ds.shape[0] + 31) // 32, dtype=torch.int32, device=dev)
            rates = []
            for layout in (api.LAYOUT_CWBVH, api.LAYOUT_BVH):
                if layout == api.LAYOUT_CWBVH:
                    for e in (before, after):
                        api.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_CWBVH))
                for rep in range(args.reps):
                    for arm, e in (("before", before), ("after", after)) if rep % 2 == 0 else (("after", after), ("before", before)):
                        e.layout = layout
                        cs = rate(lambda: (wc.copy_(dc), e.Intersect(wc), e.IsOccluded(ds, bits)), dc.shape[0] + ds.shape[0], 3)
                        df = rate(lambda: (wd.copy_(dd), e.Intersect(wd)), dd.shape[0], 3)
                        rates.append({"layout": "CWBVH" if layout == api.LAYOUT_CWBVH else "BVH", "arm": arm, "rep": rep,
                                      "camera_shadow_grays": cs, "diffuse_grays": df})
            row["rates"] = rates
            rows[name] = row
            del before, after, step
            torch.cuda.empty_cache()
        out["scenes"][label] = {"tris": int(v.shape[0] // 3), "trees": rows}
        print(json.dumps({label: out["scenes"][label]}), flush=True)
    s = json.dumps(out)
    print(s)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "optimize_perf.json"), "w").write(s + "\n")


if __name__ == "__main__":
    main()
