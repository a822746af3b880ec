"""The host model of tests/handle_model.py on its own: the named and seeded sequences of tests/test_handle_sequences_gpu.py run through
the model alone, and after every step each model tree is well formed, the closest hits of the handles the step changed are a brute force over
their current soup, and their closest-point walk is the brute force of the same rules.  A model bug fails here, before any device is involved."""
import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import rays as R, scenes
from tests import closest_oracle as co, handle_model as hm, util


class HostPool(hm.Pool):
    def __init__(self):
        super().__init__()
        lo, hi = scenes.scene_bounds(np.concatenate([m[0] for m in self.meshes]))
        rng = np.random.default_rng(5)
        c = (lo + hi) * 0.5
        O = (c + (rng.random((3, 3)) - 0.5) * (hi - lo) * 1.5).astype(np.float32)
        D = (c + (rng.random((3, 3)) - 0.5) * (hi - lo) * 0.3 - O).astype(np.float32)
        self.rays = R.make_rays(O, D)
        self.q = np.zeros((48, 4), np.float32)
        self.q[:, :3] = c + (rng.random((48, 3)) - 0.5) * (hi - lo) * 1.2
        self.q[:, 3] = np.inf

    def check(self):
        for m in self.models:
            if m.tree is None:
                continue
            t = m.tree
            util.check_tree((t.nodes, t.prim_idx, m.idx_count), t.verts.shape[0] // 3)
            if m.kind != "blas" or m not in self.touched:
                continue                 # the brute forces below run on the handles the step changed
            assert np.array_equal(t.verts.view(np.uint32), m.verts.view(np.uint32)), self.trace()
            got = self.rays.copy()
            t.intersect(got)
            v = m.verts
            for i in range(self.rays.shape[0]):
                best = np.float32(1e30)
                for j in range(v.shape[0] // 3):
                    hit, tt, _, _ = portpy.tri_test(self.rays["O"][i], self.rays["D"][i], v[3 * j, :3], v[3 * j + 1, :3], v[3 * j + 2, :3], best)
                    if hit:
                        best = np.float32(tt)
                assert got["t"][i] == best, f"handle {m.name}: ray {i} t {got['t'][i]} != brute {best}\n" + self.trace()
            walk = co.walk(t.nodes, t.prim_idx, v, self.q)
            brute = co.brute(t.nodes, t.prim_idx, v, self.q)
            assert np.array_equal(walk.view(np.uint32), brute.view(np.uint32)), f"handle {m.name}\n" + self.trace()
            if m.cw is not None and m.cw_built is not None:
                assert m.cw_built.shape == t.nodes.shape, "the kept collapse belongs to a tree of the same shape"


@pytest.mark.parametrize("name", list(hm.NAMED))
def test_named(name):
    p = HostPool()
    hm.NAMED[name](p)


def test_named_codes():
    """the codes the model gives the calls the named sequences exist for"""
    p = HostPool()
    p.step("build", 0, "Build")
    p.step("convert_cw", [0])
    assert p.step("prepare", 0, "sdf") == hm.OK
    p.step("convert_cw", [0])
    assert hm.query_code(p.models[0], "sdf") == hm.OK, "a re-conversion leaves the tree and the vertices: the table stays valid"
    p.step("refit", [0], 1, False, 1)
    assert hm.query_code(p.models[0], "sdf") == hm.STATE
    p.step("build", 1, "BuildHQ")
    p.step("convert_cw", [1])
    assert p.step("refit", [1], 1, False, 2) == hm.STATE
    assert p.step("refit", [0], 1, True, 3, "V") == hm.STATE, "an indexed refit of a handle that kept no indices"
    assert p.step("build_batch", [0, 0], "Build") == hm.ARG
    p.step("tlas", 2, [0, 1], 4)
    assert p.models[2].tlas_walk_code(hm.CW) == hm.OK
    assert p.step("prepare", 2, "wn") == hm.UNSUPPORTED
    assert p.step("optimize", 2, 2) == (hm.STATE, 0)
    p.step("convert_cw", [1])
    assert p.models[2].tlas_walk_code(hm.BVH) == hm.STATE
    assert len(p.log) == 14


@pytest.mark.parametrize("seed", hm.SEEDS)
def test_random(seed):
    p = HostPool()
    hm.seq_random(p, seed)
