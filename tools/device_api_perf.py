"""Camera rays then shadow rays over bench.py's default workload (Bistro, BuildHQ -> CWBVH, 2048 x 2048 x 16 camera rays, one shadow
ray per camera ray towards the point light), in two arms:

  (a) tbvh_intersect_device, a shadow-record kernel, tbvh_occluded_device - three launches, the hits and the shadow records in HBM;
  (b) one kernel of the caller's (tests/device_api_consumer.cu k_camera_shadow) that traces the camera ray with
      tbvh::intersect_cwbvh, builds the shadow ray in registers and calls tbvh::isoccluded_cwbvh.

Both arms build the shadow ray with the same device routine (device_api_consumer.cu shadow_ray), and their occlusion bits and shadow
records must be byte-identical before any time is reported.  After warm-up the arms alternate, each timed with CUDA events around
its launches only (the copy of the camera records that arm (a) traces in place is made before the start event).  Prints one JSON
line with the card name and power limit read in the same run.

  python tools/device_api_perf.py [--res 2048] [--reps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import bench  # noqa: E402  (the workload's scene, camera, light and epsilon)
from tinybvh_b200 import _lib, api, build, rays as R, scenes  # noqa: E402


def consumer(tmp):
    so = os.path.join(tmp, "consumer.so")
    subprocess.check_call([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + os.path.join(REPO, "include"),
                           "-Xcompiler", "-fPIC", "-shared", os.path.join(REPO, "tests", "device_api_consumer.cu"), "-o", so])
    L = C.CDLL(so)
    vp, u32, i32, f32 = C.c_void_p, C.c_uint32, C.c_int, C.c_float
    L.dc_camera_shadow_async.argtypes = [_lib.DeviceView, i32, i32, vp, vp, vp, u32, f32, f32, f32, f32, vp]
    L.dc_shadow_records_async.argtypes = [vp, vp, u32, f32, f32, f32, f32, vp]
    return L


def gpu_card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True).strip()
    except Exception as e:   # the number is reported without it rather than not at all
        return f"unknown ({e})"


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", default="bistro")
    ap.add_argument("--res", type=int, default=2048, help="camera rays = res * res * 16")
    ap.add_argument("--reps", type=int, default=10, help="timed repetitions of each arm, alternating")
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if api.device_count() == 0:
        raise SystemExit("device_api_perf: no CUDA device (there is no CPU measurement)")
    verts, label = scenes.load_scene(args.scene)
    cw = api.BVH8_CWBVH().BuildHQ(verts)
    view = cw.device_view(api.LAYOUT_CWBVH)
    eye, vdir = bench.camera_for(args.scene, verts)
    cam_h = R.primary_rays(eye, vdir, args.res, args.res, 16)
    n = cam_h.shape[0]
    cam = torch.from_numpy(np.ascontiguousarray(cam_h.view(np.uint8).reshape(-1, 128)[:, :64])).cuda()
    del cam_h
    light, eps = bench.light_for(args.scene, verts), bench.shadow_eps(verts)
    lx, ly, lz = map(float, light)
    traced = torch.empty_like(cam)
    sh_a, sh_b = torch.empty_like(cam), torch.empty_like(cam)
    words = (n + 31) // 32
    bits_a, bits_b = (torch.empty(words, dtype=torch.int32, device="cuda") for _ in range(2))
    s = torch.cuda.current_stream()
    st = C.c_void_p(s.cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())
    Lb = _lib.lib()
    with tempfile.TemporaryDirectory() as tmp:
        L = consumer(tmp)

        def arm_a():
            _lib.check(Lb.tbvh_intersect_device(cw.h, api.LAYOUT_CWBVH, p(traced), 64, None, n, st))
            assert L.dc_shadow_records_async(p(traced), p(sh_a), n, lx, ly, lz, eps, st) == 0
            _lib.check(Lb.tbvh_occluded_device(cw.h, api.LAYOUT_CWBVH, p(sh_a), 64, p(bits_a), n, st))

        def arm_b():
            bits_b.zero_()
            assert L.dc_camera_shadow_async(view, 1, 1, p(cam), p(sh_b), p(bits_b), n, lx, ly, lz, eps, st) == 0

        def timed(arm):
            traced.copy_(cam)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            arm()
            e1.record(s)
            e1.synchronize()
            return e0.elapsed_time(e1)

        timed(arm_a), timed(arm_b)
        torch.cuda.synchronize()
        if not (torch.equal(bits_a, bits_b) and torch.equal(sh_a, sh_b)):
            raise SystemExit("device_api_perf: the arms disagree (occlusion bits or shadow records); no time is reported")
        for _ in range(args.warmup):
            timed(arm_a), timed(arm_b)
        ta, tb = [], []
        for _ in range(args.reps):
            ta.append(timed(arm_a))
            tb.append(timed(arm_b))
        assert torch.equal(bits_a, bits_b)
    ma, mb = float(np.median(ta)), float(np.median(tb))
    print(json.dumps({"gpu": gpu_card(), "scene": label, "tris": int(verts.shape[0] // 3), "camera_rays": n, "shadow_rays": n,
                      "occluded": int(np.unpackbits(bits_a.cpu().numpy().view(np.uint8)).sum()),
                      "a_batch_ms_median": ma, "a_batch_ms": ta, "b_fused_ms_median": mb, "b_fused_ms": tb, "b_over_a": mb / ma,
                      "a": "tbvh_intersect_device + shadow-record kernel + tbvh_occluded_device",
                      "b": "one kernel: tbvh::intersect_cwbvh, shadow ray in registers, tbvh::isoccluded_cwbvh"}))


if __name__ == "__main__":
    main()
