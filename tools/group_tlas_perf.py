"""An instanced scene on a device group, on the GPU: `python tools/group_tlas_perf.py [--out DIR] [--reps 5] [--rays 1048576]`.

Scenes: the 32-BLAS scene of tools/tlas_frame_perf.py at 1,000 and 100,000 instances, and workload a of tools/build_batch_perf.py (1,000
BLASes, two instances each).  The BLASes are BVH8_CWBVH objects (BVH and CWBVH layouts both travel).  Per scene:
  - bytes: what one replicate copies to each device that is not the source's (computed from the handles' sizes) - the first replicate,
    a rigid frame (new transforms: the TLAS arrays only) and a deforming frame (refit_batch( keep_layouts = 1 ): every BLAS again);
  - wall (host clock around the call, which ends in a device synchronise) and device time (the call's own ms) of a first replicate on a
    fresh group, a rigid-frame refresh and a deforming-frame refresh: medians over --reps repetitions after a warm-up, the three kinds
    alternated in order;
  - tbvh_launch_count() per call;
  - closest-hit traversal of one host ray batch through the group (tbvh_group_intersect, CWBVH layout) against the source handle's own
    tbvh_intersect on the same rays, wall medians, and whether the hits are identical.
The card's name and power limit come from nvidia-smi (read-only).  On a one-GPU machine the group is device 0 twice, so the copies
stay within HBM; over NVLink they would cross the link.  Needs a CUDA device.  Prints one JSON line (and writes it to DIR when given)."""
import argparse
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
from tinybvh_b200 import api, build, rays as R, scenes  # noqa: E402
from build_batch_perf import gpu_card, stats, workload  # noqa: E402
from tlas_frame_perf import transforms  # noqa: E402


def devices():
    n = api.device_count()
    return list(range(n)) if n > 1 else [0, 0]


def copy_bytes(t, blas):
    """(first, rigid, deforming) bytes one replicate of TLAS t sends to each destination device"""
    ti = t.info()
    tlas = max(ti.used_nodes, 2) * 32 + ti.idx_count * 4 + ti.prim_count * 80 + len(blas) * 48
    per = 0
    for b in {id(b): b for b in blas}.values():
        i = b.info()
        per += max(i.used_nodes, 2) * 32 + i.idx_count * 48 + (i.used_blocks // 5) * 160 + i.cwbvh_tri_count * 48
    return tlas + per, tlas, tlas + per


def timed(fn):
    l0, t0 = api.launch_count(), time.perf_counter()
    ms = fn()
    return (time.perf_counter() - t0) * 1e3, ms, api.launch_count() - l0


def run_scene(meshes, n_inst, reps, n_rays, seed):
    blas = api.build_batch([api.BVH8_CWBVH() for _ in meshes], meshes)
    m = len(blas)
    inst = np.zeros(n_inst, api.BLAS_INSTANCE)
    inst["blasIdx"], inst["mask"] = np.arange(n_inst) % m, 0xFFFF
    spread = 4.0 * n_inst ** (1 / 3)
    inst["transform"] = transforms(n_inst, seed, spread)
    t = api.TLAS()
    t.Rebuild(inst, blas, api.LAYOUT_CWBVH)
    out = {"blasses": m, "instances": n_inst, "group_devices": devices()}
    first_b, rigid_b, deform_b = copy_bytes(t, blas)
    out["bytes_per_device"] = {"first": first_b, "rigid": rigid_b, "deforming": deform_b}
    g = api.Group(devices())
    res = {"first": [], "rigid": [], "deforming": []}
    frame = 0
    for rep in range(-1, reps):   # rep -1 warms up
        order = ["first", "rigid", "deforming"]
        order = order[rep % 3:] + order[:rep % 3] if rep >= 0 else order
        for kind in order:
            frame += 1
            if kind == "first":
                g.close()
                g = api.Group(devices())
                r = timed(lambda: g.replicate(t))
            else:
                if kind == "deforming":
                    api.refit_batch(blas, meshes, keep_layouts=1)
                inst["transform"] = transforms(n_inst, seed + frame, spread)
                t.Rebuild(inst)
                r = timed(lambda: g.replicate(t))
            if rep >= 0:
                res[kind].append(r)
    for kind, xs in res.items():
        out[kind] = {"wall_ms": stats([x[0] for x in xs]), "device_ms": stats([x[1] for x in xs]), "launches": sorted({x[2] for x in xs})}
    # traversal through the group against the source handle, same rays
    lo, hi = inst["aabbMin"].min(0), inst["aabbMax"].max(0)
    rays = R.primary_rays(*R.bounds_camera(lo, hi, "outside"), 1024, n_rays // 1024, 1)[:n_rays]
    grp_rays, src_rays = g.empty_rays(rays.shape[0], R.RAY_DTYPE), g.empty_rays(rays.shape[0], R.RAY_DTYPE)   # both page-locked
    walls = {"group": [], "source": []}
    same = True
    for rep in range(-1, reps):
        for which in (("group", "source") if rep & 1 else ("source", "group")):
            if which == "group":
                grp_rays[:] = rays
                t0 = time.perf_counter()
                g.Intersect(grp_rays)
            else:
                src_rays[:] = rays
                t0 = time.perf_counter()
                t.Intersect(src_rays)
            if rep >= 0:
                walls[which].append((time.perf_counter() - t0) * 1e3)
        same = same and grp_rays.tobytes() == src_rays.tobytes()
    out["traversal"] = {"rays": int(rays.shape[0]), "layout": "CWBVH", "group_wall_ms": stats(walls["group"]), "source_wall_ms": stats(walls["source"]),
                        "identical": bool(same), "hits": int((src_rays["t"] < 1e30).sum())}
    g.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rays", type=int, default=1 << 20)
    a = ap.parse_args()
    if api.device_count() < 1:
        sys.exit("group_tlas_perf: no CUDA device (a copy time is a GPU measurement)")
    build.build()
    result = {"card": gpu_card(), "group_devices": devices(), "scenes": {}}
    frame_meshes = [scenes.procedural_scene(300 + 150 * k, 40 + k) for k in range(32)]
    for n in (1000, 100000):
        result["scenes"][f"tlas_frame_32x{n}"] = run_scene(frame_meshes, n, a.reps, a.rays, 900)
    result["scenes"]["workload_a_1000x2000"] = run_scene(workload("a"), 2000, a.reps, a.rays, 1900)
    text = json.dumps(result)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "group_tlas_perf.json"), "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
