"""Winding numbers through the C++ shim: harness/winding_number_b200.cpp compiles against the C-ABI (CPU) and runs on the GPU - 0 and 1
outside and inside a sphere, about 0.5 at the centre of an open hemisphere, 2 in the overlap of two spheres, and the refusal of a stale
table after a refit."""
import os
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def compile_harness(out_dir):
    from tinybvh_b200 import build
    build.build()
    out = os.path.join(str(out_dir), "winding_number_b200")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"),
                           os.path.join(REPO, "harness", "winding_number_b200.cpp"), "-L" + os.path.join(REPO, "tinybvh_b200"), "-ltinybvh_b200",
                           "-Wl,-rpath," + os.path.join(REPO, "tinybvh_b200"), "-o", out])
    return out


def test_winding_number_harness_compiles_and_links(tmp_path):
    assert os.path.isfile(compile_harness(tmp_path))


@pytest.mark.gpu
def test_winding_number_harness_runs(gpu, tmp_path):
    r = subprocess.run([compile_harness(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 failures" in r.stdout, r.stdout
