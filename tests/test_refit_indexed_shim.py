"""The C++ side of indexed refits: BVH::Refit and RefitBatch of objects built with Build( vertices, indices, primCount ) compile against
the C-ABI (CPU), and harness/refit_indexed_b200.cpp runs on the GPU - every tree refitted from its moved vertex array equal to a twin
built and refitted from the flat triangle soup."""
import os
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def compile_harness(out_dir):
    from tinybvh_b200 import build
    build.build()
    out = os.path.join(str(out_dir), "refit_indexed_b200")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "harness", "refit_indexed_b200.cpp"),
                           "-L" + os.path.join(REPO, "tinybvh_b200"), "-ltinybvh_b200", "-Wl,-rpath," + os.path.join(REPO, "tinybvh_b200"), "-o", out])
    return out


def test_refit_indexed_harness_compiles_and_links(tmp_path):
    assert os.path.isfile(compile_harness(tmp_path))


@pytest.mark.gpu
def test_refit_indexed_harness_runs(gpu, tmp_path):
    r = subprocess.run([compile_harness(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 trees differ" in r.stdout, r.stdout
