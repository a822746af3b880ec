"""The host restatement of the proximity queries (tests/closest_oracle.c, DESIGN.md §4.9), without a GPU: the per-triangle function
against fp64 geometry, its barycentric range, the brute force over every reference against the pruned walk on trees of every builder and
of the uploaded-tree families, the sphere bit against the closest point, and the path bound down every path."""
import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import scenes
from tests import closest_oracle as co, ploc_oracle, util


def fp64_closest(p, a, b, c):
    """distance from p to the triangle (a, b, c) in fp64: the plane point when it lies inside, else the nearest of the three segments"""
    p, a, b, c = (np.asarray(x, np.float64)[:, :3] for x in (p, a, b, c))

    def seg(s, t):
        d = t - s
        dd = (d * d).sum(1)
        w = np.clip(np.where(dd > 0, ((p - s) * d).sum(1) / np.where(dd > 0, dd, 1), 0), 0, 1)
        return np.linalg.norm(p - (s + w[:, None] * d), axis=1)

    best = np.minimum(np.minimum(seg(a, b), seg(a, c)), seg(b, c))
    n = np.cross(b - a, c - a)
    nn = (n * n).sum(1)
    ok = nn > 1e-30 * np.maximum(((b - a) ** 2).sum(1) * ((c - a) ** 2).sum(1), 1e-300)
    nz = np.where(ok, nn, 1)
    t = ((p - a) * n).sum(1) / nz
    q = p - t[:, None] * n
    inside = ok.copy()
    for s, e in ((a, b), (b, c), (c, a)):
        inside &= (np.cross(e - s, q - s) * n).sum(1) >= 0
    face = np.abs(t) * np.sqrt(nz)
    return np.where(inside, np.minimum(face, best), best)


def triangle_cases(seed=5):
    """(v0, e1, e2, points, label) per kind: random, slivers, collinear, zero-area, coincident triangles; points on vertices, edges and
    faces, off the surface and far away"""
    rng = np.random.default_rng(seed)
    n = 4000
    kinds = {}
    a = rng.normal(size=(n, 3)) * 3
    kinds["random"] = (a, a + rng.normal(size=(n, 3)), a + rng.normal(size=(n, 3)))
    d = rng.normal(size=(n, 3))
    kinds["sliver"] = (a, a + d, a + d * rng.uniform(0.2, 0.8, (n, 1)) + rng.normal(size=(n, 3)) * 1e-5)
    kinds["collinear"] = (a, a + d, a + d * rng.uniform(-2, 2, (n, 1)))
    kinds["zero_area"] = (a, a + d, a.copy())
    kinds["coincident"] = (a, a.copy(), a.copy())
    for name, (A, B, C) in kinds.items():
        A, B, C = (np.asarray(x, np.float32) for x in (A, B, C))
        e1, e2 = B - A, C - A                  # the leaf record, in fp32 as the engine writes it
        b, c = A.astype(np.float64) + e1, A.astype(np.float64) + e2
        w = rng.dirichlet((1, 1, 1), n)
        t = rng.uniform(0, 1, (n, 1))
        pts = {
            "vertex": np.choose(rng.integers(0, 3, n)[:, None], [A, b, c]),
            "edge": np.choose(rng.integers(0, 3, n)[:, None], [A + t * e1, A + t * e2, b + t * (c - b)]),
            "face": w[:, :1] * A + w[:, 1:2] * b + w[:, 2:] * c,
            "off": A + rng.normal(size=(n, 3)) * 2,
            "far": A + rng.normal(size=(n, 3)) * 1e4,
        }
        for pk, P in pts.items():
            yield A, e1, e2, np.asarray(P, np.float32), f"{name}/{pk}"


DEGENERATE = ("sliver", "collinear", "zero_area", "coincident")


def test_triangle_distance_matches_fp64():
    """sqrt(d2_raw) is the fp64 distance to the record's triangle within 2e-6 of the inputs' magnitude (fp32 rounding of ap and of the
    products).  Only on the degenerate kinds - slivers, collinear, zero-area and coincident triangles, whose face weights carry no
    digits and whose nearest edge point stands in - may it be off by up to twice the triangle's width (its height over the longest
    edge) besides.  The point v0 + u e1 + v e2 lies at that distance within the same bound; u, v are finite, >= 0, not -0 and
    u + v <= 1 in fp32."""
    for A, e1, e2, P, label in triangle_cases():
        d2, u, v = co.triangles(P, A, e1, e2)
        b, c = A.astype(np.float64) + e1, A.astype(np.float64) + e2
        want = fp64_closest(P, A, b, c)
        scale = np.abs(np.concatenate([P, A, e1, e2], 1)).max(1) + 1e-30
        tol = 2e-6 * scale
        if label.split("/")[0] in DEGENERATE:
            e1d, e2d = e1.astype(np.float64), e2.astype(np.float64)
            longest = np.maximum(np.maximum(np.linalg.norm(e1d, axis=1), np.linalg.norm(e2d, axis=1)), np.linalg.norm(e2d - e1d, axis=1))
            tol = tol + 2 * np.linalg.norm(np.cross(e1d, e2d), axis=1) / np.where(longest > 0, longest, 1)
        err = np.abs(np.sqrt(d2.astype(np.float64)) - want)
        assert (err <= tol).all(), f"{label}: worst error {(err / tol).max():.3g} x the tolerance"
        assert np.isfinite(u).all() and np.isfinite(v).all(), label
        assert (u >= 0).all() and (v >= 0).all() and ((u + v) <= np.float32(1)).all(), label
        assert not np.signbit(u).any() and not np.signbit(v).any(), f"{label}: a -0 weight"
        # the closest point itself: v0 + u e1 + v e2 is at the returned distance
        q = A.astype(np.float64) + u[:, None].astype(np.float64) * e1 + v[:, None].astype(np.float64) * e2
        dq = np.linalg.norm(P.astype(np.float64) - q, axis=1)
        assert (np.abs(dq - want) <= tol).all(), f"{label}: the point v0 + u e1 + v e2 is off by {(np.abs(dq - want) / tol).max():.3g} x the tolerance"


def test_degenerate_rules():
    """zero-length edges give their start point; a zero-area face takes the nearest clamped edge point, ties to AB"""
    z = np.zeros((1, 3), np.float32)
    _, u, v = co.triangles(np.array([[1, 1, 1]], np.float32), z, z, z)
    assert (u[0], v[0]) == (0, 0)
    # b == c: BC has zero length; the point beyond b along e1 lands on B
    e = np.array([[1, 0, 0]], np.float32)
    d2, u, v = co.triangles(np.array([[2, 0, 0]], np.float32), z, e, e)
    assert d2[0] == 1 and (u[0], v[0]) == (1, 0)


def queries_for(v, rng, n=1500, r_kinds=True):
    """near-surface samples, points uniform in twice the box, far points and points on vertices, with a mix of r_max"""
    tri = v.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    lo, hi = tri.reshape(-1, 3).min(0), tri.reshape(-1, 3).max(0)
    ext = float((hi - lo).max())
    k = rng.integers(0, tri.shape[0], n)
    w = rng.dirichlet((1, 1, 1), n)
    near = (w[:, :, None] * tri[k]).sum(1) + rng.normal(size=(n, 3)) * 0.01 * ext
    mid, half = (lo + hi) / 2, (hi - lo)
    uni = mid + rng.uniform(-1, 1, (n, 3)) * half
    far = mid + rng.normal(size=(n // 4, 3)) * 50 * ext
    vert = tri[rng.integers(0, tri.shape[0], n // 4), rng.integers(0, 3, n // 4)]
    p = np.concatenate([near, uni, far, vert]).astype(np.float32)
    q = np.zeros((p.shape[0], 4), np.float32)
    q[:, :3] = p
    q[:, 3] = np.inf
    if r_kinds:
        sel = rng.integers(0, 7, p.shape[0])
        r = np.choose(sel, [np.full(p.shape[0], np.inf), np.zeros(p.shape[0]), np.full(p.shape[0], 1e-6 * ext),
                            rng.uniform(0, 0.05 * ext, p.shape[0]), rng.uniform(0, 0.5 * ext, p.shape[0]),
                            np.full(p.shape[0], -1.0), np.full(p.shape[0], np.nan)]).astype(np.float32)
        q[:, 3] = r
        q[:3, 0] = np.nan
    return q


def builder_trees(v):
    """(label, nodes, primIdx) of every builder's tree over v"""
    out = []
    o = portpy.PortBVH(v)
    out.append(("Build", o.nodes, o.prim_idx))
    a = portpy.PortBVH(v, avx=True)
    out.append(("BuildAVX", a.nodes, a.prim_idx))
    hn, hi, _ = portpy.build_hq(v)
    out.append(("BuildHQ", hn, hi))
    pn, pi, _, _ = ploc_oracle.build(v)
    out.append(("BuildPLOC", pn, pi))
    return out


def shrunk(nodes, seed, frac=0.3):
    """the same tree with a seeded share of its interior boxes shrunk towards their centres: child boxes stick out of their parents"""
    nodes = nodes.copy()
    rng = np.random.default_rng(seed)
    inner = np.nonzero((nodes["triCount"] == 0) & (np.arange(nodes.shape[0]) != 1))[0]
    pick = inner[rng.random(inner.shape[0]) < frac]
    c = (nodes["aabbMin"][pick] + nodes["aabbMax"][pick]) / 2
    nodes["aabbMin"][pick] = c + (nodes["aabbMin"][pick] - c) * 0.5
    nodes["aabbMax"][pick] = c + (nodes["aabbMax"][pick] - c) * 0.5
    return nodes


def dag(nodes, seed):
    """the same tree turned into a DAG, as tbvh_upload_bvh accepts one: a seeded interior node X of the root's left subtree takes the child
    pair of a seeded interior node Y of the right subtree (and Y's box), so Y's children are reached on two paths with different path
    bounds, and X's old subtree is no longer reached"""
    nodes = nodes.copy()
    rng = np.random.default_rng(seed)

    def inner_under(r):
        out, st = [], [r]
        while st:
            x = st.pop()
            if nodes["triCount"][x] == 0:
                out.append(x)
                st += [int(nodes["leftFirst"][x]), int(nodes["leftFirst"][x]) + 1]
        return out

    root_lf = int(nodes["leftFirst"][0])
    xs, ys = inner_under(root_lf)[1:], inner_under(root_lf + 1)[1:]
    x, y = int(rng.choice(xs)), int(rng.choice(ys))
    nodes["leftFirst"][x] = nodes["leftFirst"][y]
    nodes["aabbMin"][x], nodes["aabbMax"][x] = nodes["aabbMin"][y], nodes["aabbMax"][y]
    return nodes


def check_same(nodes, idx, v, q, label):
    b = co.brute(nodes, idx, v, q)
    w = co.walk(nodes, idx, v, q)
    assert np.array_equal(b.view(np.uint32), w.view(np.uint32)), f"{label}: pruned walk differs from the brute force"
    bits = co.brute(nodes, idx, v, q, any_=True)
    assert np.array_equal(co.walk(nodes, idx, v, q, any_=True), bits), f"{label}: overlap bits of the walk differ"
    found = co.record_prims(b) != co.NO_PRIM
    got = np.unpackbits(bits.view(np.uint8), bitorder="little")[: q.shape[0]].astype(bool)
    assert np.array_equal(got, found), f"{label}: sphere bit is not 'closest point within r finds a triangle'"
    return b


@pytest.mark.parametrize("ntris", [1, 7, 2000])
def test_brute_force_equals_pruned_walk(ntris):
    v = scenes.procedural_scene(ntris, 11 + ntris)
    rng = np.random.default_rng(ntris)
    q = queries_for(v, rng, n=600)
    for label, nodes, idx in builder_trees(v):
        b = check_same(nodes, idx, v, q, f"{label}-{ntris}")
        miss = co.record_prims(b) == co.NO_PRIM
        assert np.array_equal(b[miss, 0].view(np.uint32), q[miss, 3].view(np.uint32)), "miss records carry r_max"
        assert not miss[3:][np.isinf(q[3:, 3])].any(), "an unbounded query always finds a triangle"


def test_failed_split_sbvh_brute_force_equals_pruned_walk():
    """an SBVH whose spatial splits fail: leaves built from stale idxTmp words need not hold their triangles"""
    from tests.test_build_hq_shapes import fail_scene, fail_scene_hq
    v = fail_scene("snapped3k_q4")
    nodes, idx = fail_scene_hq("snapped3k_q4")[:2]
    check_same(nodes, idx, v, queries_for(v, np.random.default_rng(6), n=800), "snapped3k_q4")


def family(src, fam):
    """(nodes, primIdx) of util's uploaded-tree family `fam`, or "shrunk" (child boxes outside their parents), or "dag" (a slot reached
    on two paths)"""
    if fam == "shrunk":
        return shrunk(src[0], 3), src[1]
    if fam == "dag":
        return dag(src[0], 3), src[1]
    return util.family_tree(src, fam, 17)[:2]


@pytest.mark.parametrize("fam", util.FAMILIES + ["shrunk", "dag"])
def test_families_brute_force_equals_pruned_walk(fam):
    v = scenes.procedural_scene(3000, 71)
    src = util.source_tree(v, "BuildHQ" if fam in ("A1", "DB") else "Build")
    nodes, idx = family(src, fam)
    check_same(nodes, idx, v, queries_for(v, np.random.default_rng(9), n=500), fam)


def leaf_bounds_and_distances(nodes, idx, v, p):
    """for one point: every reached leaf's path bound P (the oracle's box arithmetic) and the fp64 squared distance to the nearest of
    its triangles"""
    P = co.node_bounds(nodes, p)
    leaves = np.nonzero((P >= 0) & (nodes["triCount"] > 0))[0]
    tri = v.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    n = tri.shape[0]
    d2 = fp64_closest(np.repeat(p[None, :3], n, 0), tri[:, 0], tri[:, 1], tri[:, 2]) ** 2
    lf, cnt = nodes["leftFirst"][leaves].astype(np.int64), nodes["triCount"][leaves].astype(np.int64)
    owner = np.repeat(np.arange(leaves.shape[0]), cnt)
    pos = np.concatenate([np.arange(a, a + c) for a, c in zip(lf, cnt)])
    near = np.full(leaves.shape[0], np.inf)
    np.minimum.at(near, owner, d2[idx[pos]])
    return P[leaves].astype(np.float64), near


@pytest.mark.parametrize("fam", ["Build", "BuildAVX", "BuildPLOC"] + util.FAMILIES + ["dag"])
def test_path_bound_is_a_lower_bound(fam):
    """Where every leaf box holds its triangles (the binned and PLOC builders, and the uploaded families and DAG made from the binned
    tree), the path bound of a leaf - the largest box bound on its path, the least over its paths - never exceeds the true squared
    distance to any of its triangles (fp64, within fp32 rounding), so the clamp d2 = fmaxf( d2_raw, P ) changes nothing but rounding
    and pruning by P never drops the nearest triangle."""
    v = scenes.procedural_scene(3000, 71)
    if fam == "BuildPLOC":
        nodes, idx = ploc_oracle.build(v)[:2]
    elif fam == "BuildAVX":
        a = portpy.PortBVH(v, avx=True)
        nodes, idx = a.nodes, a.prim_idx
    else:
        src = util.source_tree(v, "Build")
        nodes, idx = (src[0], src[1]) if fam == "Build" else family(src, fam)
    scale2 = float(np.abs(v[:, :3]).max()) ** 2
    for p in queries_for(v, np.random.default_rng(4), n=40, r_kinds=False):
        P, near = leaf_bounds_and_distances(nodes, idx, v, p)
        s2 = max(scale2, float(np.abs(p[:3]).max()) ** 2)
        assert (P <= near * (1 + 1e-5) + 1e-10 * s2).all(), f"{fam}: a path bound exceeds the distance to its leaf's triangles"
        assert (P > 0).any(), f"{fam}: the bounds prune nothing"


def test_path_bound_raises_leaves_outside_their_boxes():
    """A tree whose boxes do not hold their triangles (interior boxes shrunk): some leaf's path bound exceeds its triangles' true
    distance, so the clamp raises those references - the case DESIGN §4.9 rule 3 defines rather than excludes."""
    v = scenes.procedural_scene(3000, 71)
    src = util.source_tree(v, "Build")
    nodes, idx = family(src, "shrunk")
    raised = 0
    for p in queries_for(v, np.random.default_rng(4), n=40, r_kinds=False):
        P, near = leaf_bounds_and_distances(nodes, idx, v, p)
        raised += int((P > near * (1 + 1e-3)).sum())
    assert raised > 0


def test_python_query_rows():
    """(n, 4) rows are {x, y, z, r} records used as they are; a radius argument beside them, or none with (n, 3) points, is an error"""
    from tinybvh_b200 import api
    q = np.array([[1, 2, 3, 4], [5, 6, 7, np.inf]], np.float32)
    assert np.array_equal(api._np_queries(q, None), q)
    r = api._np_queries(q[:, :3], 0.5)
    assert np.array_equal(r[:, :3], q[:, :3]) and (r[:, 3] == 0.5).all()
    assert np.array_equal(api._np_queries(q[:, :3], q[:, 3])[:, 3], q[:, 3])
    with pytest.raises(api.TbvhError):
        api._np_queries(q, np.inf)
    with pytest.raises(api.TbvhError):
        api._np_queries(q[:, :3], None)
