"""Scenes on which BuildHQ's spatial splits fail often (tiny_bvh.h:2939: every fragment ends up on one side, and the leaf is
built from whatever idxTmp holds at the node's old range - words an ancestor's partition left there, or zeros), in small nodes
and in nodes of hundreds of fragments.  The GPU builder reproduces those leaves only if what a failed node reads depends on its
ancestors alone, whichever kernel and group size processes it (tests/test_build_hq_shapes_gpu.py).  Here, on the CPU: the
scenes keep that point (failed and stale leaves, in big nodes, no -0) and the restatement equals the reference on them."""
import ctypes as C
import functools

import numpy as np
import pytest

from oracle import portpy, refpy
from tinybvh_b200 import scenes
from tests import util

# name -> (builder, arguments)
FAIL_SCENES = {
    "snapped3k_q4": ("snapped", 3000, 100, 4),
    "snapped20k_q4": ("snapped", 20000, 101, 4),
    "snapped70k_q4": ("snapped", 70000, 102, 4),
    "snapped70k_q1": ("snapped", 70000, 104, 1),
    "snapped200k_q4": ("snapped", 200000, 103, 4),
    "lattice10k_k3": ("lattice", 10000, 7, 3),
    "lattice20k_k5": ("lattice", 20000, 9, 5),
}


@functools.lru_cache(maxsize=None)
def fail_scene(name):
    kind, n, seed, arg = FAIL_SCENES[name]
    v = util.snapped(scenes.procedural_scene(n, seed), arg) if kind == "snapped" else util.lattice_scene(n, seed, arg)
    v.setflags(write=False)
    return v


def oracle_hq(v):
    """portpy.build_hq with the restatement's failed-split diagnostics -> (nodes, primIdx, idxCount, failed leaves, failed
    leaves that read words their own partition did not write, fragment count of the largest failed node)."""
    L = portpy.lib()
    fs, fm = (C.c_uint32.in_dll(L, k) for k in ("orc_hq_failed_splits", "orc_hq_failed_max"))
    fs.value = fm.value = 0
    nodes, idx, ic = portpy.build_hq(v)
    return nodes, idx, ic, fs.value & 0xFFFF, fs.value >> 16, fm.value


@functools.lru_cache(maxsize=None)
def fail_scene_hq(name):
    return oracle_hq(fail_scene(name))


@pytest.mark.parametrize("name", list(FAIL_SCENES))
def test_scene_fails_splits_without_negative_zero(name):
    v = fail_scene(name)
    # BuildHQ's -0 tie rule is a known difference (tests/test_offatrium_gpu.py HQ_SIGNED_ZERO), not what these scenes test
    assert util.count_neg_zero(v[:, :3]) == 0
    _, _, _, failed, stale, largest = fail_scene_hq(name)
    assert failed > 0 and stale > 0, f"{name}: {failed} failed splits, {stale} stale"
    assert largest > 0


def test_some_scene_fails_in_a_node_above_the_warp_kernel_limit():
    """hq_small is clamped to 256: a failed node above that is processed by the level phase under every setting."""
    big = {name: fail_scene_hq(name)[5] for name in FAIL_SCENES}
    assert max(big.values()) > 256, big


def test_failed_split_diagnostics_do_not_change_the_tree():
    v = fail_scene("snapped3k_q4")
    a = oracle_hq(v)
    b = portpy.build_hq(v)
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1]) and a[2] == b[2]
    assert a[3:] == oracle_hq(v)[3:], "the diagnostics are reset by the caller and counted per build"


@pytest.mark.skipif(not refpy.available(), reason="oracle/_ref (the compiled reference) not built")
@pytest.mark.parametrize("name", list(FAIL_SCENES))
def test_port_build_hq_matches_reference_on_failing_scenes(name):
    v = fail_scene(name)
    ref = refpy.RefBVH(v, mode=2, threaded=False)
    nodes, idx, idx_count = fail_scene_hq(name)[:3]
    assert np.array_equal(nodes.view(np.uint32), ref.nodes.view(np.uint32))
    assert np.array_equal(idx, ref.prim_idx[: idx.shape[0]]) and idx.shape[0] == int(ref.nodes["triCount"].sum())
    assert idx_count == ref.idx_count
