"""The frame of an animated two-level scene, both ways, on the GPU: `python tools/tlas_frame_perf.py --out DIR [--sizes 1000,100000,1000000]`.

Host records: harness/tlas_frame_b200.cpp is compiled and run with --time at every size - per frame RefitBatch of the BLASes and new
transforms, then the TLAS by (a) a compiled loop of tbvh_instance_update and tbvh_build_tlas (the shim's Build) and (b) one
tbvh_build_tlas_update (BuildUpdated), alternating which goes first; it reports wall time around each (every call ends in a device
synchronise), the kernel launches and build_ms of each, and whether records, TLAS nodes, primIdx and the hits of a ray batch are identical.
Device records: the same frame from a CUDA torch tensor of records through api.TLAS.Rebuild, against Rebuild from a NumPy copy of the
same records: wall time, launches, build_ms and a byte comparison of records and TLAS.  The card's name and power limit come from
nvidia-smi (read-only).  Needs a CUDA device.  Writes DIR/tlas_frame_perf.json and prints it."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
from tinybvh_b200 import api, build, scenes  # noqa: E402
from build_batch_perf import gpu_card  # noqa: E402

LINE = re.compile(r"frame (-?\d+): (\d+) instances, (\d+) blasses; Update loop \+ Build ([\d.]+) ms wall, (\d+) launches, build_ms ([\d.]+); "
                  r"BuildUpdated ([\d.]+) ms wall, (\d+) launches, build_ms ([\d.]+); (\d+) of (\d+) rays hit; (\w+)")


def host_records(exe, n, m):
    r = subprocess.run([exe, "--time", str(n), str(m)], capture_output=True, text=True, timeout=1200)
    frames = []
    for g in LINE.findall(r.stdout):
        if int(g[0]) >= 0:   # frame -1 warms up
            frames.append({"loop_wall_ms": float(g[3]), "loop_launches": int(g[4]), "loop_build_ms": float(g[5]),
                           "one_call_wall_ms": float(g[6]), "one_call_launches": int(g[7]), "one_call_build_ms": float(g[8]), "identical": g[11] == "identical"})
    return {"exit_code": r.returncode, "frames": frames}


def transforms(n, seed, spread):
    rng = np.random.default_rng(seed)
    a, b = rng.random(n) * 6.28, rng.random(n) * 6.28
    t = np.zeros((n, 4, 4), np.float32)
    t[:, 0, 0], t[:, 0, 1], t[:, 0, 2] = np.cos(a) * np.cos(b), -np.sin(b), np.sin(a) * np.cos(b)
    t[:, 1, 0], t[:, 1, 1], t[:, 1, 2] = np.cos(a) * np.sin(b), np.cos(b), np.sin(a) * np.sin(b)
    t[:, 2, 0], t[:, 2, 2] = -np.sin(a), np.cos(a)
    t[:, :3, :3] *= (0.5 + rng.random((n, 1, 3))).astype(np.float32)
    t[:, :3, 3] = (rng.random((n, 3)) - 0.5) * spread
    t[:, 3, 3] = 1
    return t.reshape(n, 16)


def device_records(n, m, frames=3):
    import torch
    blas = [api.BVH().Build(scenes.procedural_scene(300 + 150 * k, 40 + k)) for k in range(m)]
    inst = np.zeros(n, api.BLAS_INSTANCE)
    inst["blasIdx"], inst["mask"] = np.arange(n) % m, 0xFFFF
    dev_t, host_t = api.TLAS(), api.TLAS()
    out = []
    for f in range(-1, frames):   # frame -1 warms up
        inst["transform"] = transforms(n, 900 + f, 4.0 * n ** (1 / 3))
        host = inst.copy()
        d = torch.from_numpy(inst.view(np.uint8).reshape(n, 192)).cuda()
        torch.cuda.synchronize()
        res = {}
        for which in (("device", "host") if f & 1 else ("host", "device")):
            l0, t0 = api.launch_count(), time.perf_counter()
            (dev_t.Rebuild(d, blas) if which == "device" else host_t.Rebuild(host, blas))
            res[which + "_wall_ms"] = (time.perf_counter() - t0) * 1e3   # the call synchronises the engine stream before it returns
            res[which + "_launches"] = api.launch_count() - l0
            res[which + "_build_ms"] = (dev_t if which == "device" else host_t).info().build_ms
        same = d.cpu().numpy().tobytes() == host.tobytes()
        for x, y in zip(dev_t.download(), host_t.download()):
            same = same and x.tobytes() == y.tobytes()
        res["identical"] = bool(same)
        if f >= 0:
            out.append(res)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--sizes", default="1000,100000,1000000")
    ap.add_argument("--blasses", type=int, default=32)
    a = ap.parse_args()
    if api.device_count() < 1:
        sys.exit("tlas_frame_perf: no CUDA device (a frame time is a GPU measurement)")
    build.build()
    os.makedirs(a.out, exist_ok=True)
    result = {"card": gpu_card(), "blasses": a.blasses, "sizes": {}}
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "tlas_frame_b200")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "harness", "tlas_frame_b200.cpp"),
                               "-L" + os.path.join(REPO, "tinybvh_b200"), "-ltinybvh_b200", "-Wl,-rpath," + os.path.join(REPO, "tinybvh_b200"), "-o", exe])
        for n in [int(x) for x in a.sizes.split(",")]:
            result["sizes"][str(n)] = {"host_records": host_records(exe, n, a.blasses), "device_records": device_records(n, a.blasses)}
    text = json.dumps(result, indent=1)
    with open(os.path.join(a.out, "tlas_frame_perf.json"), "w") as f:
        f.write(text)
    print(text)


if __name__ == "__main__":
    main()
