"""Times of impact between moving meshes through the C++ shim: harness/mesh_toi_b200.cpp compiles against the C-ABI (CPU) and runs on the
GPU - TimeOfImpact and ImpactPairs on triangles falling onto a plate against their double-precision first times of contact."""
import os
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def compile_harness(out_dir):
    from tinybvh_b200 import build
    build.build()
    out = os.path.join(str(out_dir), "mesh_toi_b200")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"),
                           os.path.join(REPO, "harness", "mesh_toi_b200.cpp"), "-L" + os.path.join(REPO, "tinybvh_b200"), "-ltinybvh_b200",
                           "-Wl,-rpath," + os.path.join(REPO, "tinybvh_b200"), "-o", out])
    return out


def test_mesh_toi_harness_compiles_and_links(tmp_path):
    assert os.path.isfile(compile_harness(tmp_path))


@pytest.mark.gpu
def test_mesh_toi_harness_runs(gpu, tmp_path):
    r = subprocess.run([compile_harness(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 failures" in r.stdout, r.stdout
