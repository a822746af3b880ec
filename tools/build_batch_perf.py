"""Batched builds and conversions against loops of single ones, on the GPU: `python tools/build_batch_perf.py --out DIR [--reps N]`.

Workloads (seeded, procedural):
  a  1,000 meshes, triangle counts log-uniform in [64, 20000]  (a scene of many small BLASses)
  b  16 meshes of 100k..500k triangles + 500 of 100..5,000     (a few big meshes among many small ones)
For each: a loop of tbvh_build over the meshes and one tbvh_build_batch, alternated, after a warm-up of each - host wall time around the
complete call(s), device time (sum of info.build_ms for the loop, the batch's build_ms), kernel launches, and a byte comparison of every
tree.  Then the CWBVH conversion of the same meshes' BuildAVX trees (what BVH8_CWBVH builds over): a loop of tbvh_convert( CWBVH ) per
handle and one tbvh_convert_batch, alternated - wall time (both calls end in a synchronise), launches, and a byte comparison of every
bvh8Data / bvh8Tris.  Then the one-tree path against an older build of the library (--parent-lib, when given): tbvh_build of the
Bistro-sized procedural scene and of a 150k-triangle scene, and the wall time of tbvh_convert( CWBVH ) of the Bistro-sized scene's
Build and BuildHQ trees, and the wall time of one tbvh_convert_batch( CWBVH ) of workload a's BuildAVX trees and of 200 BuildHQ trees
with a byte comparison of every handle, the two libraries alternated on the same card.  The card's name and power limit come from nvidia-smi (read-only).
The HQ arm (--arms hq, or all): on workloads a and b, a loop of tbvh_build_flavour( BuildHQ ) over the meshes against one
tbvh_build_batch_hq, alternated after a warm-up of each - wall time, device time, launches and a byte comparison of every handle's nodes
and primIdx - and, with --parent-lib, a single BuildHQ of the Bistro-sized procedural scene (the build bench.py times) in both
libraries, alternated.
Writes DIR/build_batch_perf.json and prints it."""
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
from tinybvh_b200 import _lib, api, scenes  # noqa: E402


def gpu_card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def workload(name):
    if name == "a":
        rng = np.random.default_rng(1001)
        sizes = np.exp(rng.uniform(np.log(64), np.log(20000), 1000)).astype(int)
    else:
        rng = np.random.default_rng(1002)
        sizes = np.concatenate([rng.integers(100000, 500001, 16), np.exp(rng.uniform(np.log(100), np.log(5000), 500)).astype(int)])
        sizes = sizes[rng.permutation(sizes.shape[0])]
    return [scenes.procedural_scene(int(n), 10000 + k) for k, n in enumerate(sizes)]


def stats(xs):
    xs = sorted(xs)
    return {"median": xs[len(xs) // 2], "min": xs[0], "max": xs[-1], "all": xs}


class Lib:
    """One copy of the engine library with its own context and handles (ctypes loads each path separately)."""

    def __init__(self, path):
        self.L = C.CDLL(path)
        for name, (res, args) in _lib.SYMBOLS.items():
            if hasattr(self.L, name):
                f = getattr(self.L, name)
                f.restype, f.argtypes = res, args
        self.ctx = C.c_void_p()
        self.check(self.L.tbvh_ctx_create(0, C.byref(self.ctx)))

    def check(self, rc):
        if rc != 0:
            raise RuntimeError(f"error {rc}: {self.L.tbvh_last_error().decode()}")

    def handles(self, n):
        hs = (C.c_void_p * n)()
        for k in range(n):
            h = C.c_void_p()
            self.check(self.L.tbvh_bvh_create(self.ctx, C.byref(h)))
            hs[k] = h.value
        return hs

    def info(self, h):
        i = _lib.Info()
        self.check(self.L.tbvh_bvh_info(h, C.byref(i)))
        return i

    def build(self, h, v, flavour=0):
        self.check(self.L.tbvh_build_flavour(h, v.ctypes.data, 16, v.shape[0] // 3, _lib.HOST, 1.0, 1.0, flavour))

    def download_cwbvh(self, h):
        i = self.info(h)
        d = np.zeros(i.used_blocks * 4, np.uint32)
        t = np.zeros(i.cwbvh_tri_count * 12, np.uint32)
        self.check(self.L.tbvh_download_cwbvh(h, d.ctypes.data, t.ctypes.data, _lib.HOST))
        return d, t

    def download(self, h):
        i = self.info(h)
        nodes = np.zeros(i.used_nodes * 8, np.uint32)
        idx = np.zeros(i.idx_count, np.uint32)
        self.check(self.L.tbvh_download_bvh(h, nodes.ctypes.data, idx.ctypes.data, _lib.HOST))
        return nodes, idx


def run_workload(L, meshes, reps):
    n = len(meshes)
    loop_h, batch_h = L.handles(n), L.handles(n)
    recs = (_lib.Mesh * n)(*[_lib.Mesh(v.ctypes.data, 16, 0, None, v.shape[0] // 3) for v in meshes])
    res = {"loop": {"wall_ms": [], "device_ms": [], "launches": []}, "batch": {"wall_ms": [], "device_ms": [], "launches": []}}

    def loop():
        n0 = L.L.tbvh_launch_count()
        t0 = time.perf_counter()
        for k, v in enumerate(meshes):
            L.build(loop_h[k], v)
        wall = (time.perf_counter() - t0) * 1e3
        return wall, sum(L.info(loop_h[k]).build_ms for k in range(n)), L.L.tbvh_launch_count() - n0

    def batch():
        n0 = L.L.tbvh_launch_count()
        t0 = time.perf_counter()
        L.check(L.L.tbvh_build_batch(batch_h, recs, n, _lib.HOST, 1.0, 1.0, 0))
        wall = (time.perf_counter() - t0) * 1e3
        return wall, L.info(batch_h[0]).build_ms, L.L.tbvh_launch_count() - n0

    loop(), batch()   # warm-up: first launches, allocator
    for _ in range(reps):
        for name, f in (("loop", loop), ("batch", batch)):
            w, d, l = f()
            res[name]["wall_ms"].append(w), res[name]["device_ms"].append(d), res[name]["launches"].append(l)
    same = 0
    for k in range(n):
        a, b = L.download(loop_h[k]), L.download(batch_h[k])
        same += np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    for hs in (loop_h, batch_h):
        L.check(L.L.tbvh_build_batch(hs, recs, n, _lib.HOST, 1.0, 1.0, _lib.BUILD_AVX))
    conv = {"loop": {"wall_ms": [], "launches": []}, "batch": {"wall_ms": [], "launches": []}}

    def conv_loop():
        t0 = time.perf_counter()
        for k in range(n):
            L.check(L.L.tbvh_convert(loop_h[k], _lib.LAYOUT_CWBVH))
        return (time.perf_counter() - t0) * 1e3

    def conv_batch():
        t0 = time.perf_counter()
        L.check(L.L.tbvh_convert_batch(batch_h, n, _lib.LAYOUT_CWBVH))
        return (time.perf_counter() - t0) * 1e3

    conv_loop(), conv_batch()   # warm-up
    for _ in range(reps):
        for name, f in (("loop", conv_loop), ("batch", conv_batch)):
            n0 = L.L.tbvh_launch_count()
            conv[name]["wall_ms"].append(f())
            conv[name]["launches"].append(L.L.tbvh_launch_count() - n0)
    cw_same = 0
    for k in range(n):
        a, b = L.download_cwbvh(loop_h[k]), L.download_cwbvh(batch_h[k])
        cw_same += np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    for h in list(loop_h) + list(batch_h):
        L.L.tbvh_bvh_destroy(h)
    out = {"meshes": n, "triangles": int(sum(v.shape[0] // 3 for v in meshes)), "trees_identical": int(same)}
    for name in ("loop", "batch"):
        out[name] = {k: stats(v) for k, v in res[name].items()}
    out["speedup_wall_median"] = out["loop"]["wall_ms"]["median"] / out["batch"]["wall_ms"]["median"]
    out["convert_cwbvh"] = {name: {k: stats(v) for k, v in conv[name].items()} for name in conv}
    out["convert_cwbvh"]["cwbvh_identical"] = int(cw_same)
    out["convert_cwbvh"]["speedup_wall_median"] = out["convert_cwbvh"]["loop"]["wall_ms"]["median"] / out["convert_cwbvh"]["batch"]["wall_ms"]["median"]
    return out


def run_hq_workload(L, meshes, reps):
    """a loop of BuildHQ over the meshes against one tbvh_build_batch_hq"""
    n = len(meshes)
    loop_h, batch_h = L.handles(n), L.handles(n)
    recs = (_lib.Mesh * n)(*[_lib.Mesh(v.ctypes.data, 16, 0, None, v.shape[0] // 3) for v in meshes])
    res = {"loop": {"wall_ms": [], "device_ms": [], "launches": []}, "batch": {"wall_ms": [], "device_ms": [], "launches": []}}

    def loop():
        n0 = L.L.tbvh_launch_count()
        t0 = time.perf_counter()
        for k, v in enumerate(meshes):
            L.build(loop_h[k], v, _lib.BUILD_HQ)
        wall = (time.perf_counter() - t0) * 1e3
        return wall, sum(L.info(loop_h[k]).build_ms for k in range(n)), L.L.tbvh_launch_count() - n0

    def batch():
        n0 = L.L.tbvh_launch_count()
        t0 = time.perf_counter()
        L.check(L.L.tbvh_build_batch_hq(batch_h, recs, n, _lib.HOST, 1.0, 1.0))
        wall = (time.perf_counter() - t0) * 1e3
        return wall, L.info(batch_h[0]).build_ms, L.L.tbvh_launch_count() - n0

    loop(), batch()   # warm-up
    for _ in range(reps):
        for name, f in (("loop", loop), ("batch", batch)):
            w, d, l = f()
            res[name]["wall_ms"].append(w), res[name]["device_ms"].append(d), res[name]["launches"].append(l)
    same = 0
    for k in range(n):
        a, b = L.download(loop_h[k]), L.download(batch_h[k])
        ia, ib = L.info(loop_h[k]), L.info(batch_h[k])
        same += np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and bytes(ia)[:_lib.Info.build_ms.offset] == bytes(ib)[:_lib.Info.build_ms.offset]
    for h in list(loop_h) + list(batch_h):
        L.L.tbvh_bvh_destroy(h)
    out = {"meshes": n, "triangles": int(sum(v.shape[0] // 3 for v in meshes)), "handles_identical": int(same)}
    for name in ("loop", "batch"):
        out[name] = {k: stats(v) for k, v in res[name].items()}
    out["speedup_wall_median"] = out["loop"]["wall_ms"]["median"] / out["batch"]["wall_ms"]["median"]
    return out


def one_tree_hq(libs, reps):
    """BuildHQ of the Bistro-sized procedural scene (bench.py's tree) in every library, alternated: device and wall time"""
    v = scenes.procedural_scene(2837209, 7)
    hs = {name: L.handles(1) for name, L in libs.items()}
    dev, wall = {name: [] for name in libs}, {name: [] for name in libs}
    for name, L in libs.items():
        L.build(hs[name][0], v, _lib.BUILD_HQ)   # warm-up
    for r in range(reps):
        for name, L in libs.items() if r % 2 == 0 else reversed(list(libs.items())):
            t0 = time.perf_counter()
            L.build(hs[name][0], v, _lib.BUILD_HQ)
            wall[name].append((time.perf_counter() - t0) * 1e3)
            dev[name].append(L.info(hs[name][0]).build_ms)
    trees = [L.download(hs[name][0]) for name, L in libs.items()]
    out = {"device_ms": {name: stats(x) for name, x in dev.items()}, "wall_ms": {name: stats(x) for name, x in wall.items()}}
    out["trees_identical"] = all(np.array_equal(t[0], trees[0][0]) and np.array_equal(t[1], trees[0][1]) for t in trees)
    for name, L in libs.items():
        L.L.tbvh_bvh_destroy(hs[name][0])
    return out


def one_tree(libs, reps):
    out = {}
    for label, v in (("bistro_sized_2837209", scenes.procedural_scene(2837209, 7)), ("tris_150k", scenes.procedural_scene(150000, 8))):
        hs = {name: L.handles(1) for name, L in libs.items()}
        ms = {name: [] for name in libs}
        for name, L in libs.items():
            L.build(hs[name][0], v)   # warm-up
        for _ in range(reps):
            for name, L in libs.items():
                L.build(hs[name][0], v)
                ms[name].append(L.info(hs[name][0]).build_ms)
        trees = [L.download(hs[name][0]) for name, L in libs.items()]
        out[label] = {name: stats(x) for name, x in ms.items()}
        out[label]["trees_identical"] = all(np.array_equal(t[0], trees[0][0]) and np.array_equal(t[1], trees[0][1]) for t in trees)
        for name, L in libs.items():
            L.L.tbvh_bvh_destroy(hs[name][0])
    return out


def one_tree_convert(libs, reps):
    """tbvh_convert( CWBVH ) of one big tree, wall time: the path bench.py reports as cwbvh_convert_ms_wall."""
    v = scenes.procedural_scene(2837209, 7)
    out = {}
    for label, flavour in (("bistro_sized_build", _lib.BUILD_REFERENCE), ("bistro_sized_buildhq", _lib.BUILD_HQ)):
        hs = {name: L.handles(1) for name, L in libs.items()}
        ms = {name: [] for name in libs}
        for name, L in libs.items():
            L.build(hs[name][0], v, flavour)
            L.check(L.L.tbvh_convert(hs[name][0], _lib.LAYOUT_CWBVH))   # warm-up
        for _ in range(reps):
            for name, L in libs.items():
                t0 = time.perf_counter()
                L.check(L.L.tbvh_convert(hs[name][0], _lib.LAYOUT_CWBVH))
                ms[name].append((time.perf_counter() - t0) * 1e3)
        cws = [L.download_cwbvh(hs[name][0]) for name, L in libs.items()]
        out[label] = {name: stats(x) for name, x in ms.items()}
        # bvh8Tris past the referenced records is uninitialised on an SBVH: compare bvh8Data and the records of the Build tree
        out[label]["bvh8data_identical"] = all(np.array_equal(c[0], cws[0][0]) for c in cws)
        if flavour != _lib.BUILD_HQ:
            out[label]["bvh8tris_identical"] = all(np.array_equal(c[1], cws[0][1]) for c in cws)
        for name, L in libs.items():
            L.L.tbvh_bvh_destroy(hs[name][0])
    return out


def batch_convert(libs, reps):
    """tbvh_convert_batch( CWBVH ) in one call per library, the libraries alternated: workload a's BuildAVX trees, and 200 BuildHQ trees
    (SBVHs: a batch of trees that keep no collapse)"""
    rng = np.random.default_rng(1003)
    hq = [scenes.procedural_scene(int(n), 20000 + k) for k, n in enumerate(np.exp(rng.uniform(np.log(64), np.log(20000), 200)).astype(int))]
    out = {}
    for label, meshes, flavour in (("workload_a_buildavx", workload("a"), _lib.BUILD_AVX), ("buildhq_200", hq, _lib.BUILD_HQ)):
        n = len(meshes)
        hs = {name: L.handles(n) for name, L in libs.items()}
        for name, L in libs.items():
            for k, v in enumerate(meshes):
                L.build(hs[name][k], v, flavour)
        ms = {name: [] for name in libs}
        for r in range(reps + 1):   # r = 0 warms both up
            for name, L in libs.items() if r % 2 == 0 else reversed(list(libs.items())):
                t0 = time.perf_counter()
                L.check(L.L.tbvh_convert_batch(hs[name], n, _lib.LAYOUT_CWBVH))
                if r:
                    ms[name].append((time.perf_counter() - t0) * 1e3)
        out[label] = {name: stats(x) for name, x in ms.items()}
        # bvh8Tris past the referenced records is uninitialised on an SBVH: bvh8Data only for BuildHQ
        same = 0
        for k in range(n):
            cws = [L.download_cwbvh(hs[name][k]) for name, L in libs.items()]
            same += all(np.array_equal(c[0], cws[0][0]) and (flavour == _lib.BUILD_HQ or np.array_equal(c[1], cws[0][1])) for c in cws)
        out[label]["handles_identical"] = int(same)
        out[label]["handles"] = n
        for name, L in libs.items():
            for h in hs[name]:
                L.L.tbvh_bvh_destroy(h)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for build_batch_perf.json")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parent-lib", default=None, help="libtinybvh_b200.so of an older build to compare the one-tree path with")
    ap.add_argument("--arms", choices=("all", "sah", "hq"), default="all", help="sah: the binned-SAH builds and conversions; hq: BuildHQ")
    args = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("build_batch_perf: needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    L = Lib(_lib.SO)
    result = {"card": gpu_card(), "reps": args.reps}
    libs = {"this": L}
    if args.parent_lib:
        libs = {"parent": Lib(args.parent_lib), "this": L}
    if args.arms in ("all", "sah"):
        for name in ("a", "b"):
            result[f"workload_{name}"] = run_workload(L, workload(name), args.reps)
        result["one_tree_build_ms"] = one_tree(libs, max(args.reps, 7))
        result["one_tree_convert_cwbvh_wall_ms"] = one_tree_convert(libs, max(args.reps, 7))
        result["batch_convert_cwbvh_wall_ms"] = batch_convert(libs, max(args.reps, 7))
    if args.arms in ("all", "hq"):
        for name in ("a", "b"):
            result[f"hq_workload_{name}"] = run_hq_workload(L, workload(name), args.reps)
        if args.parent_lib:
            result["one_tree_buildhq"] = one_tree_hq(libs, max(args.reps, 10))
    path = os.path.join(args.out, "build_batch_perf.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
