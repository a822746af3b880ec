"""BuildHQ under every setting that changes which kernel and group size processes a node: the switch point to the
warp-per-subtree kernel (hq_small), the largest thread-block cluster (hq_cluster) and the cluster sizing rule's fragments per CTA
and CTAs per SM (TBVH_HQ_CTA_FRAGS, TBVH_HQ_CTA_CAP).  On scenes whose spatial splits fail often, in small and in big nodes
(tests/test_build_hq_shapes.py), the tree must stay the reference's byte for byte: a failed node's leaf is read from idxTmp
words an ancestor left behind, which only holds when those words do not depend on the order nodes are processed in.  The
profile output proves each setting took effect.  Also: the SBVH's derived layouts and walks under three settings, and the
binned-SAH builder's persistent large phase (build_ctas)."""
import functools
import re

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import api, scenes
from tinybvh_b200._lib import BUILD_AVX, BUILD_REFERENCE
from tests import util
from tests.test_build_gpu import assert_same_tree
from tests.test_build_hq_gpu import assert_same_hq_tree
from tests.test_build_hq_shapes import FAIL_SCENES, fail_scene, fail_scene_hq, oracle_hq

pytestmark = pytest.mark.gpu

HQ_ENV = ("TBVH_HQ_CTA_FRAGS", "TBVH_HQ_CTA_CAP", "TBVH_HQ_PROFILE")
HQ_DEFAULTS = {"hq_small": 16, "hq_cluster": 16}
# name -> (context options, environment)
CONFIGS = {
    "defaults": ({}, {}),
    "small8": ({"hq_small": 8}, {}),
    "small17": ({"hq_small": 17}, {}),
    "small64": ({"hq_small": 64}, {}),
    "small256": ({"hq_small": 256}, {}),
    "small0": ({"hq_small": 0}, {}),          # clamps to 8
    "small1000": ({"hq_small": 1000}, {}),    # clamps to 256
    "cluster1": ({"hq_cluster": 1}, {}),      # one 256-thread CTA per node, a 70k-fragment root included
    "cluster2": ({"hq_cluster": 2}, {}),
    "cluster3": ({"hq_cluster": 3}, {}),
    "cluster12": ({"hq_cluster": 12}, {}),
    "frags1_capmax": ({}, {"TBVH_HQ_CTA_FRAGS": "1", "TBVH_HQ_CTA_CAP": "1048576"}),   # every level node gets the largest cluster
    "frags_max": ({}, {"TBVH_HQ_CTA_FRAGS": "1048576"}),                               # always one CTA
    "cap1": ({}, {"TBVH_HQ_CTA_CAP": "1"}),
    "small256_frags1": ({"hq_small": 256}, {"TBVH_HQ_CTA_FRAGS": "1"}),
    "small8_cluster16_frags1": ({"hq_small": 8, "hq_cluster": 16}, {"TBVH_HQ_CTA_FRAGS": "1"}),
}


def effective(cfg):
    """-> (switch point, largest cluster the sizing rule may pick, whether every level node gets it) of a configuration."""
    opts, env = CONFIGS[cfg]
    small = min(max(opts.get("hq_small", 16), 8), 256)
    cluster = min(max(opts.get("hq_cluster", 16), 1), 16)
    top = 1 << (cluster.bit_length() - 1)       # the sizing rule doubles from 1
    if env.get("TBVH_HQ_CTA_FRAGS") == "1048576":
        top = 1
    return small, top, env.get("TBVH_HQ_CTA_FRAGS") == "1" and env.get("TBVH_HQ_CTA_CAP") == "1048576"


@pytest.fixture
def knobs(request, monkeypatch):
    """Sets a CONFIGS entry for one test; the options live in the shared context, so the defaults always come back."""
    opts, env = CONFIGS[request.param]
    for k in HQ_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    try:
        for k, val in {**HQ_DEFAULTS, **opts}.items():
            api.set_option(k, val)
        yield request.param
    finally:
        for k, val in HQ_DEFAULTS.items():
            api.set_option(k, val)


def degenerate(name):
    if name == "identical":
        return np.tile(util.ONE_TRI, (700, 1))
    if name == "duplicates":
        base = scenes.procedural_scene(900, 13)
        return np.concatenate([base, base, base[:300]])
    # long thin triangles: long unsplitting chains
    rng = np.random.default_rng(17)
    c = rng.random((2000, 3), np.float32) * 10
    d = (rng.random((2000, 3), np.float32) - 0.5) * np.array([8, 0.05, 0.05], np.float32)
    w = (rng.random((2000, 3), np.float32) - 0.5) * 0.05
    v = np.zeros((6000, 4), np.float32)
    v[0::3, :3], v[1::3, :3], v[2::3, :3] = c - d, c + d, c + w
    return v


PROCEDURAL = {"proc255": (255, 41), "proc257": (257, 42), "proc5000": (5000, 43), "proc70000": (70000, 44)}
SCENES = list(FAIL_SCENES) + ["slivers", "identical", "duplicates"] + list(PROCEDURAL)


@functools.lru_cache(maxsize=None)
def scene_and_tree(name):
    """-> (vertices, the restatement's BuildHQ: nodes, primIdx, idxCount, failed leaves, stale, largest failed node)"""
    if name in FAIL_SCENES:
        return (fail_scene(name),) + fail_scene_hq(name)
    v = scenes.procedural_scene(*PROCEDURAL[name]) if name in PROCEDURAL else degenerate(name)
    return (v,) + oracle_hq(v)


@pytest.mark.parametrize("name", SCENES)
@pytest.mark.parametrize("knobs", list(CONFIGS), indirect=True)
def test_build_hq_matches_oracle_under_knobs(gpu, knobs, name):
    v, nodes, idx, ic = scene_and_tree(name)[:4]
    assert_same_hq_tree(api.BVH().BuildHQ(v), nodes, idx, ic, f"{name} {knobs}")


LEVEL = re.compile(r"hq-level\s+(\d+) nodes\s+(\d+) nct\s+(\d+) max\s+(\d+):")
TOTALS = re.compile(r"hq-profile failed_splits (\d+) small_roots (\d+)")


def profiled_build(monkeypatch, capfd, v, level):
    """BuildHQ with TBVH_HQ_PROFILE=level -> (handle, [(nodes, nct, largest node) per level], failed_splits, small_roots)"""
    monkeypatch.setenv("TBVH_HQ_PROFILE", str(level))
    capfd.readouterr()
    try:
        e = api.BVH().BuildHQ(v)
    finally:
        monkeypatch.delenv("TBVH_HQ_PROFILE")
    err = capfd.readouterr().err
    levels = [tuple(int(x) for x in m.groups()[1:]) for m in LEVEL.finditer(err)]
    totals = TOTALS.findall(err)
    assert len(totals) == 1, err[-2000:]
    return e, levels, int(totals[0][0]), int(totals[0][1])


@pytest.mark.parametrize("knobs", list(CONFIGS), indirect=True)
def test_knobs_take_effect(gpu, knobs, monkeypatch, capfd):
    """The level phase's cluster sizes and node sizes as the profile prints them, and the failed-split count: the setting is the
    one the build ran with, and profiling does not change the tree."""
    v, nodes, idx, ic, failed = scene_and_tree("snapped70k_q1")[:5]
    small, top, every_level = effective(knobs)
    e, levels, got_failed, roots = profiled_build(monkeypatch, capfd, v, 2)
    assert_same_hq_tree(e, nodes, idx, ic, f"profiled {knobs}")
    assert got_failed == failed
    assert levels and roots > 0
    nct = [c for _, c, _ in levels]
    assert all(c & (c - 1) == 0 for c in nct), nct
    assert max(nct) == top, f"{knobs}: cluster sizes {nct}, largest allowed {top}"
    if every_level:
        assert set(nct) == {top}, nct
    assert all(m > small for _, _, m in levels), f"{knobs}: a level-phase node at or below the switch point {small}"
    assert levels[0][2] == v.shape[0] // 3


def test_small_roots_follow_hq_small(gpu, monkeypatch, capfd):
    """The number of subtrees handed to the warp kernel moves with hq_small, and out-of-range values clamp to 8 and 256."""
    v, nodes, idx, ic, failed = scene_and_tree("snapped70k_q1")[:5]
    for k in HQ_ENV:
        monkeypatch.delenv(k, raising=False)
    roots = {}
    try:
        for small in (0, 8, 16, 64, 256, 1000):
            api.set_option("hq_small", small)
            e, _, got_failed, roots[small] = profiled_build(monkeypatch, capfd, v, 1)
            assert_same_hq_tree(e, nodes, idx, ic, f"hq_small {small}")
            assert got_failed == failed
    finally:
        api.set_option("hq_small", 16)
    assert roots[0] == roots[8] and roots[1000] == roots[256], roots
    assert len({roots[s] for s in (8, 16, 64, 256)}) == 4, roots


@functools.lru_cache(maxsize=None)
def layout_oracle():
    """snapped70k_q1 (failed splits in nodes of up to 350 fragments): the reference's BVH_GPU and CWBVH of its SBVH, and traced
    camera, shadow and diffuse rays."""
    v = fail_scene("snapped70k_q1")
    o = util.oracle_tree(v, 2)
    gpu_nodes = util.oracle_bvh_gpu_nodes(o)
    cw, used = util.oracle_cwbvh(v, mode=1)
    sets, bounds = util.ray_sets(v, res=64)
    traced = sets["primary"].copy()
    o.intersect(traced)
    sets.update(util.derived_sets(traced, v, bounds))
    return v, o, gpu_nodes, cw, used, sets


def same_hits(e, want_fn, rays, label):
    want, got = rays.copy(), rays.copy()
    want_fn(want), e.Intersect(got)
    assert util.compare_hits(got, want) == {"prim": 0, "t": 0, "u": 0, "v": 0}, label


@pytest.mark.parametrize("knobs", ["defaults", "small256", "cluster1"], indirect=True)
def test_derived_layouts_and_walks_under_knobs(gpu, knobs):
    v, o, gpu_nodes, cw, used, sets = layout_oracle()
    nodes, idx = o.nodes, o.prim_idx[: int(o.nodes["triCount"].sum())]
    walk = portpy.PortBVH(v, nodes=nodes, prim_idx=idx)
    b = api.BVH().BuildHQ(v)
    assert_same_hq_tree(b, nodes, idx, o.idx_count, knobs)
    g = api.BVH_GPU().BuildHQ(v)
    got = g.download()
    assert got.shape == gpu_nodes.shape and np.array_equal(got.view(np.uint32), gpu_nodes.view(np.uint32)), f"{knobs}: BVH_GPU nodes differ"
    c = api.BVH8_CWBVH().BuildHQ(v)
    d8, t8 = c.download()
    assert d8.shape == cw.nodes.shape and np.array_equal(d8.view(np.uint32), cw.nodes.view(np.uint32)), f"{knobs}: bvh8Data differs"
    assert t8.shape[0] >= used and np.array_equal(t8[:used].view(np.uint32), cw.tris[:used].view(np.uint32)), f"{knobs}: bvh8Tris differs"
    for kind, rays in sets.items():
        same_hits(b, walk.intersect, rays, f"{knobs} BVH {kind}")
        same_hits(g, walk.intersect, rays, f"{knobs} BVH_GPU {kind}")
        same_hits(c, cw.intersect, rays, f"{knobs} CWBVH {kind}")
    assert np.array_equal(b.IsOccluded(sets["shadow"]), walk.occluded(sets["shadow"])), f"{knobs}: occlusion bits"


# ---- BVH::Build / BuildAVX: the persistent large phase's CTAs per SM (build_ctas) -------------------------------------------
@functools.lru_cache(maxsize=None)
def sah_scene(n):
    v = scenes.procedural_scene(n, 60 + n % 97)
    v.setflags(write=False)
    return v


@functools.lru_cache(maxsize=None)
def sah_oracle(n, avx):
    o = portpy.PortBVH(sah_scene(n), avx=avx)
    return o.nodes, o.prim_idx


@pytest.fixture
def build_ctas():
    api.set_option("build_mode", 0)
    yield lambda value: api.set_option("build_ctas", value)
    api.set_option("build_ctas", 0)


@pytest.mark.parametrize("ctas", [1, 2, 16])
def test_build_ctas_trees_match_oracle(gpu, build_ctas, ctas):
    """16 is capped at the occupancy of the persistent kernel."""
    build_ctas(ctas)
    for n in (300000, 1000000):
        for method, avx in (("Build", False), ("BuildAVX", True)):
            assert_same_tree(getattr(api.BVH(), method)(sah_scene(n)), *sah_oracle(n, avx), f"{method} {n} build_ctas {ctas}")
    sizes = (300000, 5000, 129, 1)
    for flavour, avx in ((BUILD_REFERENCE, False), (BUILD_AVX, True)):
        got = api.build_batch([api.BVH() for _ in sizes], [sah_scene(n) for n in sizes], flavour)
        for e, n in zip(got, sizes):
            assert_same_tree(e, *sah_oracle(n, avx), f"batch {n} avx {avx} build_ctas {ctas}")


def test_build_ctas_moves_the_hand_over(gpu, build_ctas):
    """One CTA per SM makes the persistent grid smaller, so the build stays longer in the launch-per-stage levels."""
    v = sah_scene(300000)
    launches = {}
    for ctas in (0, 1):
        build_ctas(ctas)
        n0 = api.launch_count()
        e = api.BVH().Build(v)
        launches[ctas] = api.launch_count() - n0
        assert_same_tree(e, *sah_oracle(300000, False), f"build_ctas {ctas}")
    assert launches[1] > launches[0], launches
