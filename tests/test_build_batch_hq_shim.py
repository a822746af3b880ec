"""The C++ side of batched SBVH builds: tinybvh_b200::BuildBatch( .., TBVH_BUILD_HQ ) in the shim compiles against the C-ABI (CPU), and
harness/batch_b200.cpp runs on the GPU - every tree of its BuildHQ batch equal to a separate BuildHQ of its mesh."""
import subprocess

import pytest

from tests.test_build_batch_shim import compile_harness


def test_batch_hq_harness_compiles_and_links(tmp_path):
    import os
    assert os.path.isfile(compile_harness(tmp_path))


@pytest.mark.gpu
def test_batch_hq_harness_runs(gpu, tmp_path):
    r = subprocess.run([compile_harness(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 HQ trees differ" in r.stdout and " 0 HQ trees differ" in r.stdout, r.stdout
