"""The host restatement of generalized winding numbers (tests/wn_oracle.c, DESIGN.md §4.11), without a GPU: the fixed atan2 against
math.atan2, every record against an fp64 recomputation from its owned triangles, the exact walk (beta = inf) and the expansion (beta = 2,
4) against the fp64 winding number of tests/test_signed_distance.py on closed, open, overlapping, hollow, reversed and non-manifold
meshes, and ownership: SBVH references counted once, unused primIdx entries never reached, a DAG refused."""
import math

import numpy as np
import pytest

from tests import sdf_oracle as so, util, wn_oracle as wo
from tests.test_closest_point import builder_trees, dag
from tests.test_signed_distance import MESHES, cube, icosphere, join, soup, winding

ATAN2_BOUND = 3.0e-7                  # measured 2.93e-7 (the rounding of pi - a near +-pi)
EXACT_BOUND = 3.0e-6                  # beta = inf against fp64 at queries farther than 1e-3 of the extent from the surface: measured 1.80e-6
BETA_BOUND = {2.0: 0.11, 4.0: 0.017}  # the same queries: measured maxima 0.0727 (two_spheres) / 0.0114 (hollow), times 1.5


# ---- meshes: (V, F) float64 / int, outward by the right-hand rule where closed ---------------------------------------------------
def hemisphere():
    V, F = icosphere(3)
    return V, F[V[F].mean(1)[:, 2] > 0]


def open_cube():
    V, F = cube()
    return V, F[2:]


def two_spheres():
    return join(icosphere(2), icosphere(2, 1.0, (0.8, 0.0, 0.0)))


def reversed_sphere():
    V, F = icosphere(2)
    return V, F[:, ::-1].copy()


def book():
    """three quads on the edge x = 0, z in [0, 1]: a non-manifold edge shared by six triangles"""
    V = [[0, 0, 0], [0, 0, 1]]
    F = []
    for a in (0.0, 2.0, 4.0):
        V += [[np.cos(a), np.sin(a), 0], [np.cos(a), np.sin(a), 1]]
        i = len(V) - 2
        F += [(0, i, i + 1), (0, i + 1, 1)]
    return np.array(V, np.float64), np.array(F)


CASES = dict(MESHES, hemisphere=hemisphere, open_cube=open_cube, two_spheres=two_spheres, reversed=reversed_sphere, book=book)


def queries(V, F, rng, n=600):
    """uniform in 1.3 times the box, and jittered surface points"""
    V = np.asarray(V, np.float64)
    lo, hi = V.min(0), V.max(0)
    c, half, ext = (lo + hi) / 2, (hi - lo) / 2 * 1.3 + 1e-3, (hi - lo).max()
    tri = V[F]
    k = rng.integers(0, F.shape[0], n)
    w = rng.dirichlet((1, 1, 1), n)
    P = np.concatenate([c + rng.uniform(-1, 1, (n, 3)) * half, (tri[k] * w[:, :, None]).sum(1) + rng.normal(size=(n, 3)) * 0.03 * ext])
    q = np.zeros((P.shape[0], 4), np.float32)
    q[:, :3] = P
    return q


def away(V, F, q):
    """queries farther than 1e-3 of the extent from the surface"""
    d = np.abs(so.signed(soup(V, F), np.c_[q[:, :3], np.full(q.shape[0], np.inf, np.float32)])[:, 0])
    return d > 1e-3 * np.ptp(np.asarray(V, np.float64), 0).max()


def case_errors(name, beta, seed=0):
    V, F = CASES[name]()
    v = soup(V, F)
    q = queries(V, F, np.random.default_rng(seed + len(name)))
    w64 = winding(V, F, q[:, :3].astype(np.float64))
    ok = away(V, F, q)
    nodes, idx = builder_trees(v)[0][1:]
    got = wo.winding(nodes, idx, v, q, beta)
    return np.abs(got.astype(np.float64) - w64)[ok], got, w64, ok


# ---- atan2 -----------------------------------------------------------------------------------------------------------------------
def test_atan2_against_math():
    rng = np.random.default_rng(1)
    ang = np.linspace(-np.pi, np.pi, 200001)
    rad = np.exp(rng.uniform(-80, 80, ang.size))
    y, x = (np.sin(ang) * rad).astype(np.float32), (np.cos(ang) * rad).astype(np.float32)
    tiny = np.float32(1e-45) * np.arange(1, 9, dtype=np.float32)            # subnormals
    special = np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, 3e38, -3e38, 1e-38], np.float32)
    sy, sx = np.meshgrid(np.r_[special, tiny, -tiny], np.r_[special, tiny, -tiny])
    y, x = np.r_[y, sy.ravel()], np.r_[x, sx.ravel()]
    got = wo.atan2(y, x).astype(np.float64)
    want = np.array([math.atan2(float(a), float(b)) for a, b in zip(y, x)])
    # the engine's definition where libm's zero signs differ: y < 0 decides the sign, x < 0 the half plane (-0 is not < 0)
    zero = (y == 0) & ((x < 0) | ((x == 0) & np.signbit(x)) | np.signbit(y))
    want[zero] = np.where(x[zero] < 0, np.pi, 0.0)
    assert np.abs(got - want).max() <= ATAN2_BOUND, np.abs(got - want).max()
    assert wo.atan2([-0.0], [-1.0])[0] == np.float32(np.pi) and wo.atan2([0.0], [0.0])[0] == 0.0
    assert np.isnan(wo.atan2([np.nan, 1.0], [1.0, np.nan])).all()


# ---- records -----------------------------------------------------------------------------------------------------------------------
def owned_below(t, slot):
    """the prims the references under `slot` own (slot len(records) - 1: the root)"""
    nodes, S = t.nodes, t.records.shape[0] - 1
    out, st = [], [slot]
    while st:
        i = st.pop()
        n = nodes[0] if i == S else nodes[i]
        if n["triCount"]:
            o = t.own[int(n["leftFirst"]): int(n["leftFirst"]) + int(n["triCount"])]
            out += o[o != wo.NONE].tolist()
        else:
            st += [c for c in (int(n["leftFirst"]), int(n["leftFirst"]) + 1) if c != 1]
    return np.array(out, np.int64)


def check_records(nodes, idx, v, label):
    t = wo.Table(nodes, idx, v)
    assert t.flag == 0, label
    tri = wo._f4(v)[:, :3].astype(np.float64).reshape(-1, 3, 3)
    ext = np.ptp(tri.reshape(-1, 3), 0).max()
    # each triangle counts once: the owners are exactly the prims the tree reaches
    reached = owned_below(t, t.records.shape[0] - 1)
    assert np.unique(reached).shape[0] == reached.shape[0], f"{label}: a triangle owned twice"
    empty = t.records.view(np.uint32)[:, 3] == wo.NONE
    for slot in np.nonzero(~empty)[0]:
        prims = owned_below(t, int(slot))
        assert prims.size, f"{label}: slot {slot} owns nothing but is not empty"
        T = tri[prims]
        lo, hi = T.reshape(-1, 3).min(0), T.reshape(-1, 3).max(0)
        p, r = (lo + hi) / 2, np.linalg.norm(hi - lo) / 2
        a = 0.5 * np.cross(T[:, 1] - T[:, 0], T[:, 2] - T[:, 0])
        N = a.sum(0)
        M = ((T.mean(1) - p)[:, :, None] * a[:, None, :]).sum(0)
        rec = t.records[slot].astype(np.float64)
        scale = np.abs(a).sum() + 1e-30
        assert np.allclose(rec[:3], p, atol=1e-6 * ext) and abs(rec[3] - r) <= 1e-6 * ext, f"{label}: slot {slot} box"
        assert np.abs(rec[4:7] - N).max() <= 1e-5 * scale, f"{label}: slot {slot} N"
        assert np.abs(rec[7:].reshape(3, 3) - M).max() <= 1e-5 * scale * ext, f"{label}: slot {slot} M"
    return t


def test_records_of_every_builder_and_family():
    v = util.small_scene(1500, 13)
    for label, nodes, idx in builder_trees(v):
        check_records(nodes, idx, v, label)
    src = util.source_tree(v, "Build")
    for fam in util.FAMILIES:
        nodes, idx = util.family_tree(src, fam, 17)[:2]
        check_records(nodes, idx, v, fam)


# ---- the exact walk and the expansion against fp64 -------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_exact_walk_matches_fp64(name):
    err, got, w64, ok = case_errors(name, np.inf)
    assert ok.sum() > 0.5 * ok.shape[0]
    assert err.max() <= EXACT_BOUND, f"{name}: {err.max()}"
    if name in MESHES or name in ("two_spheres", "reversed"):   # closed: the classification is exact
        assert np.array_equal(got[ok] > 0.5, w64[ok] > 0.5)
    if name == "two_spheres":
        assert (np.abs(got[ok] - 2) < 1e-3).any(), "no query in the overlap"
    if name == "reversed":
        assert (got[ok] < -0.99).any()


@pytest.mark.parametrize("beta", sorted(BETA_BOUND))
@pytest.mark.parametrize("name", sorted(CASES))
def test_expansion_bound(name, beta):
    err, got, w64, ok = case_errors(name, beta)
    assert err.max() <= BETA_BOUND[beta], f"{name} beta {beta}: {err.max()}"
    if name in MESHES:
        assert np.array_equal(got[ok] > 0.5, w64[ok] > 0.5), f"{name} beta {beta}: classification"


def test_bistro_sized_soup_sample():
    """2.84 M triangles of the procedural soup: the one-leaf brute force against fp64 at a few points"""
    v = util.small_scene(2837209, 1)
    tri = v.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    rng = np.random.default_rng(3)
    lo, hi = tri.reshape(-1, 3).min(0), tri.reshape(-1, 3).max(0)
    q = np.zeros((6, 4), np.float32)
    q[:, :3] = lo + rng.random((6, 3)) * (hi - lo)
    got = wo.brute(v, q)
    F = np.arange(tri.shape[0] * 3).reshape(-1, 3)
    for i in range(q.shape[0]):
        w64 = winding(tri.reshape(-1, 3), F, q[i: i + 1, :3].astype(np.float64), chunk=1)[0]
        assert abs(float(got[i]) - w64) <= 2e-4, (i, got[i], w64)


# ---- ownership ---------------------------------------------------------------------------------------------------------------------
def soup_queries(v, rng, n=300):
    tri = wo._f4(v)[:, :3].reshape(-1, 3, 3)
    F = np.arange(tri.shape[0] * 3).reshape(-1, 3)
    return queries(tri.reshape(-1, 3).astype(np.float64), F, rng, n)


@pytest.mark.parametrize("name", ["snapped3k_q4", "lattice10k_k3", "scene3k"])
def test_sbvh_counts_split_triangles_once(name):
    """BuildHQ trees reference split triangles from several leaves (failed-split scenes included): at beta = inf they give the Build
    tree's winding numbers; a double-counted triangle would add its solid angle"""
    from tests.test_build_hq_shapes import fail_scene
    from oracle import portpy
    v = util.small_scene(3000, 13) if name == "scene3k" else fail_scene(name)
    hn, hi, _ = portpy.build_hq(v)
    assert int(hn["triCount"].sum()) > v.shape[0] // 3, "no triangle was split"
    q = soup_queries(v, np.random.default_rng(2))
    b = builder_trees(v)[0]
    want = wo.winding(b[1], b[2], v, q, np.inf)
    got = wo.winding(hn, hi, v, q, np.inf)
    assert np.abs(got - want).max() <= 1e-6, np.abs(got - want).max()


def test_uploaded_gaps_and_dag():
    v = soup(*icosphere(3))
    src = util.source_tree(v, "BuildHQ")
    q = queries(*icosphere(3), np.random.default_rng(4), n=300)
    for beta in (2.0, np.inf):
        want = wo.winding(src[0], src[1], v, q, beta)
        for fam in ("C0", "C3"):
            nodes, idx = util.family_tree(src, fam, 17)[:2]
            assert np.array_equal(wo.winding(nodes, idx, v, q, beta).view(np.uint32), want.view(np.uint32)), fam
    assert wo.Table(dag(util.source_tree(v, "Build")[0], 3), src[1], v).flag & wo.DAG


def test_nan_queries_and_one_leaf():
    V, F = icosphere(2)
    v = soup(V, F)
    q = np.array([[np.nan, 0, 0, 0], [0, 0, 0, 7], [5, 5, 5, 0]], np.float32)
    w = wo.brute(v, q)
    assert np.isnan(w[0]) and w.view(np.uint32)[0] == 0x7FFFFFFF
    assert abs(w[1] - 1) < 1e-5 and abs(w[2]) < 1e-5
