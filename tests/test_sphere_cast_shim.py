"""Sphere casts through the C++ shim: harness/sphere_cast_b200.cpp compiles against the C-ABI (CPU) and runs on the GPU - SphereCast
against a double-precision first contact over every triangle, SphereCastOccluded against SphereCast."""
import os
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def compile_harness(out_dir):
    from tinybvh_b200 import build
    build.build()
    out = os.path.join(str(out_dir), "sphere_cast_b200")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "harness", "sphere_cast_b200.cpp"),
                           "-L" + os.path.join(REPO, "tinybvh_b200"), "-ltinybvh_b200", "-Wl,-rpath," + os.path.join(REPO, "tinybvh_b200"), "-o", out])
    return out


def test_sphere_cast_harness_compiles_and_links(tmp_path):
    assert os.path.isfile(compile_harness(tmp_path))


@pytest.mark.gpu
def test_sphere_cast_harness_runs(gpu, tmp_path):
    r = subprocess.run([compile_harness(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 failures" in r.stdout, r.stdout
