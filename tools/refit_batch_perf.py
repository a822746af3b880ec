"""Batched refits against loops of single ones, on the GPU: `python tools/refit_batch_perf.py --out DIR [--reps N] [--parent-lib OLD.so]`.

Workloads: tools/build_batch_perf.py's (a: 1,000 meshes of 64..20,000 triangles; b: 16 meshes of 100k..500k triangles among 500 small
ones), BuildAVX trees.  Per frame the vertices are jittered (a new seed each frame) and every tree refitted:
  cwbvh  handles holding their CWBVH: a loop of tbvh_refit_layouts against one tbvh_refit_batch( .., keep_layouts = 1 )
  bvh    handles holding the BVH layout only: a loop of tbvh_refit against one tbvh_refit_batch( .., keep_layouts = 0 )
each from host and from device-resident (torch) vertices.  The two paths alternate; reported: host wall time around the complete call(s)
(every call ends in a synchronise), kernel launches, device time (the batch's build_ms; the loop's summed build_ms), and a byte
comparison of every handle after the last frame (BVH2, and bvh8Data / bvh8Tris where held).  With --parent-lib: tools/refit_perf.py's
frame - tbvh_refit_layouts of one Bistro-sized BVH::Build tree holding its CWBVH - and one tbvh_refit_batch( .., keep_layouts = 1 ) of
workload a's trees per frame, with this library and the older one, alternated.  The
card's name and power limit come from nvidia-smi (read-only).  Writes DIR/refit_batch_perf.json and prints it.

`--indexed` measures indexed meshes instead (DIR/refit_indexed_perf.json): welded deformed grids with the triangle counts of workloads a
and b (about two triangles per vertex), built with their indices and holding their CWBVH.  Per frame the vertices V are jittered and the
arms alternate, each refitting its own copy of the handles with keep_layouts = 1:
  indexed_host     tbvh_refit_batch_indexed from host V'
  expand_host      tbvh_refit_batch from the host soup V'[I], expanded by the caller each frame and timed with the expansion
  soup_host        tbvh_refit_batch from a soup expanded before the clock starts: the copy of 48 bytes per triangle alone
  indexed_device   tbvh_refit_batch_indexed from torch V'
  expand_device    tbvh_refit_batch from the torch soup V'[I], the torch gather timed with the call
Reported per arm: wall time around complete calls (each ends in a synchronise), device time (build_ms), launches, and the vertex bytes a
frame moves from host to device (computed: 16 per staged row); then a byte comparison of every handle across the arms."""
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
from tinybvh_b200 import _lib, api, scenes  # noqa: E402
from build_batch_perf import Lib, gpu_card, stats, workload  # noqa: E402


def jitter(v, seed):
    rng = np.random.default_rng(seed)
    w = v.copy()
    w[:, :3] += (rng.random((v.shape[0], 3), np.float32) - 0.5) * np.float32(0.01)
    return w


def run_workload(L, meshes, reps, mode, device):
    import torch
    n = len(meshes)
    keep = mode == "cwbvh"
    loop_h, batch_h = L.handles(n), L.handles(n)
    recs = (_lib.Mesh * n)(*[_lib.Mesh(v.ctypes.data, 16, 0, None, v.shape[0] // 3) for v in meshes])
    for hs in (loop_h, batch_h):
        L.check(L.L.tbvh_build_batch(hs, recs, n, _lib.HOST, 1.0, 1.0, _lib.BUILD_AVX))
        if keep:
            L.check(L.L.tbvh_convert_batch(hs, n, _lib.LAYOUT_CWBVH))
    single = L.L.tbvh_refit_layouts if keep else L.L.tbvh_refit
    res = {p: {"wall_ms": [], "device_ms": [], "launches": []} for p in ("loop", "batch")}

    def frame(seed):
        ws = [jitter(v, seed + k) for k, v in enumerate(meshes)]
        if not device:
            return ws, [w.ctypes.data for w in ws], _lib.HOST
        ts = [torch.from_numpy(w).cuda() for w in ws]
        torch.cuda.synchronize()
        return ts, [t.data_ptr() for t in ts], _lib.DEVICE

    def loop(ptrs, space):
        t0 = time.perf_counter()
        for k, v in enumerate(meshes):
            L.check(single(loop_h[k], ptrs[k], 16, v.shape[0] // 3, space))
        return (time.perf_counter() - t0) * 1e3, sum(L.info(loop_h[k]).build_ms for k in range(n))

    def batch(ptrs, space):
        rs = (_lib.Mesh * n)(*[_lib.Mesh(p, 16, 0, None, v.shape[0] // 3) for p, v in zip(ptrs, meshes)])
        t0 = time.perf_counter()
        L.check(L.L.tbvh_refit_batch(batch_h, rs, n, space, int(keep)))
        return (time.perf_counter() - t0) * 1e3, L.info(batch_h[0]).build_ms

    for r in range(reps + 1):   # frame 0 warms both paths up (first refits allocate their scratch)
        keep_alive, ptrs, space = frame(1000 * r)
        for name, f in (("loop", loop), ("batch", batch)) if r % 2 == 0 else (("batch", batch), ("loop", loop)):
            n0 = L.L.tbvh_launch_count()
            w, d = f(ptrs, space)
            if r:
                res[name]["wall_ms"].append(w), res[name]["device_ms"].append(d), res[name]["launches"].append(L.L.tbvh_launch_count() - n0)
    same = 0
    for k in range(n):
        a, b = L.download(loop_h[k]), L.download(batch_h[k])
        ok = np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        if keep:
            ca, cb = L.download_cwbvh(loop_h[k]), L.download_cwbvh(batch_h[k])
            ok = ok and np.array_equal(ca[0], cb[0]) and np.array_equal(ca[1], cb[1])
        same += ok
    for h in list(loop_h) + list(batch_h):
        L.L.tbvh_bvh_destroy(h)
    out = {"meshes": n, "triangles": int(sum(v.shape[0] // 3 for v in meshes)), "handles_identical": int(same)}
    for name in ("loop", "batch"):
        out[name] = {k: stats(v) for k, v in res[name].items()}
    out["speedup_wall_median"] = out["loop"]["wall_ms"]["median"] / out["batch"]["wall_ms"]["median"]
    return out


def one_tree(libs, reps):
    """tools/refit_perf.py's frame: tbvh_refit_layouts of one Bistro-sized BVH::Build tree with its CWBVH, wall and device time"""
    v = scenes.procedural_scene(2837209, 7)
    hs = {name: L.handles(1) for name, L in libs.items()}
    for name, L in libs.items():
        L.build(hs[name][0], v)
        L.check(L.L.tbvh_convert(hs[name][0], _lib.LAYOUT_CWBVH))
    wall = {name: [] for name in libs}
    dev = {name: [] for name in libs}
    for r in range(reps + 1):
        w = jitter(v, 50 + r)
        for name, L in libs.items() if r % 2 == 0 else reversed(list(libs.items())):
            t0 = time.perf_counter()
            L.check(L.L.tbvh_refit_layouts(hs[name][0], w.ctypes.data, 16, w.shape[0] // 3, _lib.HOST))
            if r:
                wall[name].append((time.perf_counter() - t0) * 1e3), dev[name].append(L.info(hs[name][0]).build_ms)
    outs = [(L.download(hs[name][0]), L.download_cwbvh(hs[name][0])) for name, L in libs.items()]
    out = {name: {"wall_ms": stats(wall[name]), "device_ms": stats(dev[name])} for name in libs}
    out["identical"] = all(all(np.array_equal(a, b) for a, b in zip(o[0] + o[1], outs[0][0] + outs[0][1])) for o in outs)
    for name, L in libs.items():
        L.L.tbvh_bvh_destroy(hs[name][0])
    return out


def batch_refit(libs, reps):
    """tbvh_refit_batch( .., keep_layouts = 1 ) of workload a's BuildAVX trees holding their CWBVH, host vertices, one call per library
    and frame, the libraries alternated: wall and device time, and a byte comparison of every handle after the last frame"""
    meshes = workload("a")
    n = len(meshes)
    recs = (_lib.Mesh * n)(*[_lib.Mesh(v.ctypes.data, 16, 0, None, v.shape[0] // 3) for v in meshes])
    hs = {name: L.handles(n) for name, L in libs.items()}
    for name, L in libs.items():
        L.check(L.L.tbvh_build_batch(hs[name], recs, n, _lib.HOST, 1.0, 1.0, _lib.BUILD_AVX))
        L.check(L.L.tbvh_convert_batch(hs[name], n, _lib.LAYOUT_CWBVH))
    wall = {name: [] for name in libs}
    dev = {name: [] for name in libs}
    for r in range(reps + 1):   # r = 0 warms both up
        ws = [jitter(v, 7000 + 1000 * r + k) for k, v in enumerate(meshes)]
        rs = (_lib.Mesh * n)(*[_lib.Mesh(w.ctypes.data, 16, 0, None, w.shape[0] // 3) for w in ws])
        for name, L in libs.items() if r % 2 == 0 else reversed(list(libs.items())):
            t0 = time.perf_counter()
            L.check(L.L.tbvh_refit_batch(hs[name], rs, n, _lib.HOST, 1))
            if r:
                wall[name].append((time.perf_counter() - t0) * 1e3), dev[name].append(L.info(hs[name][0]).build_ms)
    out = {name: {"wall_ms": stats(wall[name]), "device_ms": stats(dev[name])} for name in libs}
    same = 0
    for k in range(n):
        outs = [L.download(hs[name][k]) + L.download_cwbvh(hs[name][k]) for name, L in libs.items()]
        same += all(all(np.array_equal(a, b) for a, b in zip(o, outs[0])) for o in outs)
    out["handles_identical"], out["handles"] = int(same), n
    for name, L in libs.items():
        for h in hs[name]:
            L.L.tbvh_bvh_destroy(h)
    return out


def welded(p, seed):
    """a welded deformed grid of exactly p triangles (the first p of a grid of nx by ny cells, two triangles each): (vertices, indices)"""
    rng = np.random.default_rng(seed)
    nx = max(1, int(np.ceil(np.sqrt(p / 2))))
    ny = -(-p // (2 * nx))
    y, x = np.mgrid[0:ny + 1, 0:nx + 1].astype(np.float32)
    v = np.zeros((x.size, 4), np.float32)
    o = rng.random(3, np.float32) * 40
    v[:, 0], v[:, 1] = o[0] + x.ravel() * 0.05, o[1] + y.ravel() * 0.05
    v[:, 2] = o[2] + np.sin(x.ravel() * 0.2) * np.cos(y.ravel() * 0.3)
    a = (np.arange(ny)[:, None] * (nx + 1) + np.arange(nx)[None, :]).ravel()
    i = np.stack([a, a + 1, a + nx + 1, a + 1, a + nx + 2, a + nx + 1], 1).reshape(-1, 3)[:p]
    return v, np.ascontiguousarray(i.reshape(-1), np.uint32)


def run_indexed(L, name, reps):
    import torch
    meshes = [welded(v.shape[0] // 3, 20000 + k) for k, v in enumerate(workload(name))]
    n = len(meshes)
    arms = ("indexed_host", "expand_host", "soup_host", "indexed_device", "expand_device")
    hs = {a: L.handles(n) for a in arms}
    recs = (_lib.Mesh * n)(*[_lib.Mesh(v.ctypes.data, 16, v.shape[0], i.ctypes.data, i.shape[0] // 3) for v, i in meshes])
    for a in arms:
        L.check(L.L.tbvh_build_batch(hs[a], recs, n, _lib.HOST, 1.0, 1.0, _lib.BUILD_AVX))
        L.check(L.L.tbvh_convert_batch(hs[a], n, _lib.LAYOUT_CWBVH))
    idx_t = [torch.from_numpy(i.astype(np.int64)).cuda() for _, i in meshes]
    res = {a: {"wall_ms": [], "device_ms": [], "launches": []} for a in arms}

    def refit(a, ptrs, space, indexed):
        rs = (_lib.Mesh * n)(*[_lib.Mesh(p, 16, v.shape[0] if indexed else 0, None, i.shape[0] // 3) for p, (v, i) in zip(ptrs, meshes)])
        L.check((L.L.tbvh_refit_batch_indexed if indexed else L.L.tbvh_refit_batch)(hs[a], rs, n, space, 1))

    for r in range(reps + 1):   # r = 0 warms every arm up (first refits allocate their scratch)
        ws = [jitter(v, 3000 + 1000 * r + k) for k, (v, _) in enumerate(meshes)]
        soups = [np.take(w, i, axis=0) for w, (_, i) in zip(ws, meshes)]
        wt = [torch.from_numpy(w).cuda() for w in ws]
        torch.cuda.synchronize()

        def indexed_host():
            refit("indexed_host", [w.ctypes.data for w in ws], _lib.HOST, True)

        def expand_host():
            s = [np.take(w, i, axis=0) for w, (_, i) in zip(ws, meshes)]
            refit("expand_host", [x.ctypes.data for x in s], _lib.HOST, False)

        def soup_host():
            refit("soup_host", [x.ctypes.data for x in soups], _lib.HOST, False)

        def indexed_device():
            refit("indexed_device", [t.data_ptr() for t in wt], _lib.DEVICE, True)

        def expand_device():
            s = [torch.index_select(t, 0, i) for t, i in zip(wt, idx_t)]
            torch.cuda.synchronize()   # device-space inputs must be complete before the call reads them
            refit("expand_device", [x.data_ptr() for x in s], _lib.DEVICE, False)

        fns = dict(zip(arms, (indexed_host, expand_host, soup_host, indexed_device, expand_device)))
        for a in arms[r % len(arms):] + arms[: r % len(arms)]:
            n0 = L.L.tbvh_launch_count()
            t0 = time.perf_counter()
            fns[a]()
            wall = (time.perf_counter() - t0) * 1e3
            if r:
                res[a]["wall_ms"].append(wall), res[a]["device_ms"].append(L.info(hs[a][0]).build_ms), res[a]["launches"].append(L.L.tbvh_launch_count() - n0)
    same = 0
    for k in range(n):
        outs = [L.download(hs[a][k]) + L.download_cwbvh(hs[a][k]) for a in arms]
        same += all(all(np.array_equal(x, y) for x, y in zip(o, outs[0])) for o in outs)
    for a in arms:
        for h in hs[a]:
            L.L.tbvh_bvh_destroy(h)
    rows = sum(v.shape[0] for v, _ in meshes)
    tris = sum(i.shape[0] // 3 for _, i in meshes)
    h2d = {"indexed_host": rows * 16, "expand_host": tris * 48, "soup_host": tris * 48, "indexed_device": 0, "expand_device": 0}
    out = {"meshes": n, "triangles": int(tris), "vertices": int(rows), "handles_identical": int(same)}
    for a in arms:
        out[a] = {k: stats(v) for k, v in res[a].items()}
        out[a]["h2d_vertex_bytes_per_frame"] = int(h2d[a])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for refit_batch_perf.json")
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--parent-lib", default=None, help="libtinybvh_b200.so of an older build to compare the single refit with")
    ap.add_argument("--indexed", action="store_true", help="indexed meshes: tbvh_refit_batch_indexed against flat soups (refit_indexed_perf.json)")
    args = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("refit_batch_perf: needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    L = Lib(_lib.SO)
    result = {"card": gpu_card(), "reps": args.reps}
    if args.indexed:
        for name in ("a", "b"):
            result[f"workload_{name}_indexed"] = run_indexed(L, name, args.reps)
        path = os.path.join(args.out, "refit_indexed_perf.json")
        with open(path, "w") as f:
            json.dump(result, f, indent=1)
        print(json.dumps(result, indent=1))
        return
    for name in ("a", "b"):
        meshes = workload(name)
        for mode in ("cwbvh", "bvh"):
            for device in (False, True):
                result[f"workload_{name}_{mode}_{'device' if device else 'host'}"] = run_workload(L, meshes, args.reps, mode, device)
    if args.parent_lib:
        libs = {"parent": Lib(args.parent_lib), "this": L}
        result["one_tree_refit_layouts"] = one_tree(libs, max(args.reps, 9))
        result["batch_refit_layouts"] = batch_refit(libs, max(args.reps, 9))
    path = os.path.join(args.out, "refit_batch_perf.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
