"""The host restatement of the sphere casts (tests/sweep_oracle.c, DESIGN.md §4.16), without a GPU: the per-triangle first contact against
an independent fp64 reference (bisection on the convex distance along the sweep), analytic contacts, r = 0 against the fp64 ray crossing,
the 2^k, 2^m and -0 invariances bit for bit, translated scenes, axis-aligned sweeps, the pruned walk against the brute force over every
tree family, and zero-length sweeps against the sphere-overlap bits."""
import numpy as np
import pytest

from tinybvh_b200 import api, scenes
from tests import closest_oracle as co, sweep_oracle as so, util
from tests.test_closest_point import builder_trees, family, fp64_closest
from tests.test_intersect_all_fp64 import solve64

EPS = 2e-6          # of M, the largest relative coordinate of the case (DESIGN.md §4.16, accuracy)
EPS_DEGENERATE = 2e-5   # the same on flat caps (the sliver kind), collinear, zero-area and coincident triangles, besides twice their width (measured: 1.3e-5)
ULPS_T = 4          # fp32 ulps of t beyond the bracket: the rounding of t itself
T_RAY = 6e-6        # r = 0: |t - t64| bound, of M / |D| (measured: 5.4e-6)


def fp64_first(c, D, tmax, A, B, Cc, rho, iters=200):
    """T64(rho): the first t in [0, tmax] with dist( c + t D, triangle ) <= rho in fp64, NaN where there is none (and for rho < 0).  The
    distance is convex in t: a ternary search finds its minimum on [0, tmax], a bisection on [0, t_min] the first crossing."""
    c, D, A, B, Cc = (np.asarray(x, np.float64)[:, :3] for x in (c, D, A, B, Cc))
    tmax, rho = np.asarray(tmax, np.float64), np.asarray(rho, np.float64)
    dist = lambda t: fp64_closest(c + t[:, None] * D, A, B, Cc)
    lo, hi = np.zeros_like(tmax), tmax.copy()
    for _ in range(iters):
        a, b = lo + (hi - lo) / 3, hi - (hi - lo) / 3
        fa, fb = dist(a), dist(b)
        lo, hi = np.where(fa <= fb, lo, a), np.where(fa <= fb, b, hi)
    tmin = (lo + hi) / 2
    dmin = np.minimum(dist(tmin), np.minimum(dist(np.zeros_like(tmax)), dist(tmax)))
    tmin = np.where(dist(tmax) <= dmin, tmax, tmin)
    ok = (dmin <= rho) & (rho >= 0)
    a, b = np.zeros_like(tmax), tmin.copy()
    for _ in range(iters // 2):
        m = (a + b) / 2
        inside = dist(m) <= rho
        a, b = np.where(inside, a, m), np.where(inside, m, b)
    t = np.where(dist(np.zeros_like(tmax)) <= rho, 0.0, b)
    return np.where(ok, t, np.nan)


def magnitude(q, A, e1, e2):
    """M: the largest relative coordinate of each case - c - v0, c + tmax D - v0, the edges, r"""
    c, D = q[:, :3].astype(np.float64), q[:, 4:7].astype(np.float64)
    tm = q[:, 7].astype(np.float64)[:, None]
    r0, r1 = c - A, c + tm * D - A
    return np.max(np.abs(np.concatenate([r0, r1, e1, e2, e2 - e1, q[:, 3:4]], 1)), 1)


def width(A, e1, e2):
    """a triangle's height over its longest edge in fp64 (0 for collinear and coincident corners)"""
    e = [np.asarray(x, np.float64) for x in (e1, e2, np.asarray(e2, np.float64) - e1)]
    longest = np.max([np.linalg.norm(x, axis=1) for x in e], 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(longest > 0, np.linalg.norm(np.cross(e[0], e[1]), axis=1) / np.where(longest > 0, longest, 1), 0.0)


def check_fp64(q, A, e1, e2, label, eps=EPS, M=None, degenerate=False):
    """the rules of DESIGN.md §4.16's accuracy paragraph on one batch of (query, triangle) rows; returns the contact mask.  degenerate:
    flat caps (a corner within 1e-5 of the opposite edge), collinear, zero-area and coincident triangles, whose normal carries no
    reliable digits at any corner: delta = EPS_DEGENERATE M plus twice
    the triangle's width."""
    hit, t, u, v = so.triangles(q, A, e1, e2)
    A64 = A.astype(np.float64)
    B, Cc = A64 + e1, A64 + e2
    M = magnitude(q, A64, e1.astype(np.float64), e2.astype(np.float64)) if M is None else M
    delta = eps * M if not degenerate else EPS_DEGENERATE * M + 2 * width(A, e1, e2)
    r = q[:, 3].astype(np.float64)
    tmax = q[:, 7].astype(np.float64)
    lo = fp64_first(q[:, :3], q[:, 4:7], tmax, A64, B, Cc, r + delta)
    hi = fp64_first(q[:, :3], q[:, 4:7], tmax, A64, B, Cc, r - delta)
    slack = ULPS_T * 2.0 ** -23 * np.abs(t.astype(np.float64)) + 1e-12   # t itself is an fp32 number
    bad_miss = ~hit & ~np.isnan(hi)
    assert not bad_miss.any(), f"{label}: {int(bad_miss.sum())} misses where T64(r - delta) exists, first {np.nonzero(bad_miss)[0][:5]}"
    bad_hit = hit & np.isnan(lo)
    assert not bad_hit.any(), f"{label}: {int(bad_hit.sum())} contacts where T64(r + delta) is none, first {np.nonzero(bad_hit)[0][:5]}"
    upper = np.where(np.isnan(hi), tmax, hi)
    bad_t = hit & ((t < lo - slack) | (t > upper + slack))
    assert not bad_t.any(), f"{label}: {int(bad_t.sum())} times outside [T64(r + delta), T64(r - delta)], first {np.nonzero(bad_t)[0][:5]}: " \
        f"{t[bad_t][:3]} vs {lo[bad_t][:3]} .. {upper[bad_t][:3]}"
    assert (u[hit] >= 0).all() and (v[hit] >= 0).all() and (np.float32(u[hit]) + np.float32(v[hit]) <= 1).all(), f"{label}: contact point outside"
    p = A64 + u[:, None].astype(np.float64) * e1 + v[:, None].astype(np.float64) * e2
    centre = q[:, :3].astype(np.float64) + t[:, None].astype(np.float64) * q[:, 4:7].astype(np.float64)
    d = np.linalg.norm(centre - p, axis=1)
    at0 = hit & (t == 0)
    moving = hit & (t > 0)
    assert (d[at0] <= r[at0] + delta[at0]).all(), f"{label}: a t = 0 contact point farther than r"
    off = moving & (np.abs(d - r) > delta)
    assert not off.any(), f"{label}: {int(off.sum())} contact points not within r +- delta of the centre, worst {np.max(np.abs(d - r)[off] / M[off])}"
    return hit


def unit(x):
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def sweep_cases(seed=3, n=3000):
    """(A, e1, e2, q, label): random, sliver (a flat cap: the third corner within 1e-5 of the segment of the other two), collinear,
    zero-area and coincident triangles under random, grazing, nearly parallel and
    face-parallel sweeps (just inside and just outside r)"""
    rng = np.random.default_rng(seed)
    a = rng.normal(size=(n, 3)) * 3
    d = rng.normal(size=(n, 3))
    kinds = {
        "random": (a, a + rng.normal(size=(n, 3)), a + rng.normal(size=(n, 3))),
        "sliver": (a, a + d, a + d * rng.uniform(0.2, 0.8, (n, 1)) + rng.normal(size=(n, 3)) * 1e-5),
        "collinear": (a, a + d, a + d * rng.uniform(-2, 2, (n, 1))),
        "zero_area": (a, a + d, a.copy()),
        "coincident": (a, a.copy(), a.copy()),
    }
    for name, (A, B, C) in kinds.items():
        A, B, C = (np.asarray(x, np.float32) for x in (A, B, C))
        e1, e2 = B - A, C - A
        A64, b, c = A.astype(np.float64), A.astype(np.float64) + e1, A.astype(np.float64) + e2
        w = rng.dirichlet((1, 1, 1), n)
        X = w[:, :1] * A64 + w[:, 1:2] * b + w[:, 2:] * c                 # a target on the triangle
        r = rng.uniform(0, 1, n) * np.where(rng.random(n) < 0.2, 0.0, 1.0)
        dirs = unit(rng.normal(size=(n, 3)))
        # random: from a random start towards the target, the displacement as D with tmax 1.5
        start = X + rng.normal(size=(n, 3)) * 4
        yield A, e1, e2, so.queries(start, (X - start) * rng.uniform(0.5, 1.5, (n, 1)), r, 1.5), f"{name}/random"
        # unit directions with tmax a distance, passing the target at an offset of about r (grazing)
        side = unit(np.cross(dirs, rng.normal(size=(n, 3))))
        off = X + side * (r * (1 + rng.uniform(-1e-3, 1e-3, n)))[:, None]
        yield A, e1, e2, so.queries(off - dirs * 5, dirs, r, 10.0), f"{name}/grazing"
        # nearly parallel to the first edge
        ed = unit(e1.astype(np.float64) + rng.normal(size=(n, 3)) * 1e-4 + (np.abs(e1).sum(1) == 0)[:, None])
        yield A, e1, e2, so.queries(X - ed * 5 + side * 0.5 * r[:, None], ed, r, 10.0), f"{name}/edge-parallel"
        # parallel to the face at heights just inside and just outside r
        nrm = np.cross(e1.astype(np.float64), e2.astype(np.float64))
        ok = np.linalg.norm(nrm, axis=1) > 1e-6
        nrm = np.where(ok[:, None], nrm, rng.normal(size=(n, 3)))
        nh = unit(nrm)
        inplane = unit(np.cross(nh, rng.normal(size=(n, 3))))
        h = r * (1 + np.where(rng.random(n) < 0.5, -1, 1) * 1e-4) + 1e-3
        yield A, e1, e2, so.queries(X + nh * h[:, None] - inplane * 5, inplane, h * 0 + r + 1e-3, 10.0), f"{name}/face-parallel"


@pytest.mark.parametrize("kind", ["random", "sliver", "collinear", "zero_area", "coincident"])
def test_triangle_matches_fp64(kind):
    for A, e1, e2, q, label in sweep_cases():
        if label.startswith(kind + "/"):
            hit = check_fp64(q, A, e1, e2, label, degenerate=kind != "random")
            if kind == "random" and label.endswith("random"):
                assert 0.2 < hit.mean() < 0.98, f"{label}: contact rate {hit.mean()}"


def needle_cases(aspect, seed=11, n=2000):
    """(A, e1, e2, q, label, normal): long thin triangles of length 100 and base width `aspect` x 100 (apex angle about `aspect`
    radians, well conditioned: the largest angle is near 90 degrees), randomly placed and oriented, in all three vertex rotations, under
    head-on sweeps (along the normal, unit D) and oblique ones (displacement D, tmax 1) aimed at interior points with barycentrics >= 0.1,
    at r = 0, 0.1 and 0.4 of the width, twice the width and 1"""
    rng = np.random.default_rng(seed)
    L, h = 100.0, aspect * 100.0
    rot = np.linalg.qr(rng.normal(size=(n, 3, 3)))[0]
    base = np.array([[0, 0, 0], [L, -h / 2, 0], [L, h / 2, 0]])
    P = np.einsum("nij,kj->nki", rot, base) + rng.normal(size=(n, 1, 3)) * 50
    P = P.astype(np.float32)
    nrm = rot[:, :, 2]
    w = rng.dirichlet((1, 1, 1), n) * 0.7 + 0.1
    width = h
    r = np.choose(rng.integers(0, 5, n), [np.zeros(n), np.full(n, 0.1 * width), np.full(n, 0.4 * width), np.full(n, 2 * width), np.ones(n)])
    side = np.where(rng.random(n) < 0.5, -1.0, 1.0)[:, None]
    for k in range(3):
        V = np.roll(P, -k, axis=1)
        A = V[:, 0]
        e1, e2 = V[:, 1] - A, V[:, 2] - A
        X = np.einsum("nk,nkd->nd", np.roll(w, -k, axis=1), V.astype(np.float64))
        dist = rng.uniform(2, 20, n)
        start = X + side * nrm * dist[:, None]
        yield A, e1, e2, so.queries(start, -side * nrm, r, 40.0), f"aspect {aspect:g}, rotation {k}, head-on", nrm
        tang = np.cross(nrm, rng.normal(size=(n, 3)))
        start = X + side * nrm * dist[:, None] + tang * rng.uniform(-1, 1, (n, 1))
        yield A, e1, e2, so.queries(start, (X - start) * 1.5, r, 1.0), f"aspect {aspect:g}, rotation {k}, oblique", nrm


@pytest.mark.parametrize("aspect", [1e-3, 1e-4, 1e-5])
def test_needles(aspect):
    """long thin, well-conditioned triangles: a sweep aimed at an interior point always touches, in every vertex rotation and at every
    r, within the fp64 bracket at 2e-6 M (no width term); r = 0 gives the fp64 plane crossing within T_RAY M / |D|"""
    for A, e1, e2, q, label, nrm in needle_cases(aspect):
        hit = check_fp64(q, A, e1, e2, label)
        assert hit.all(), f"{label}: {int((~hit).sum())} sweeps through the face report no contact"
        _, t, _, _ = so.triangles(q, A, e1, e2)
        z = q[:, 3] == 0
        c, D = q[z, :3].astype(np.float64), q[z, 4:7].astype(np.float64)
        n64 = np.cross(e1[z].astype(np.float64), e2[z].astype(np.float64))
        t64 = ((A[z].astype(np.float64) - c) * n64).sum(1) / (D * n64).sum(1)
        M = magnitude(q[z], A[z].astype(np.float64), e1[z].astype(np.float64), e2[z].astype(np.float64))
        err = np.abs(t[z] - t64) / (M / np.linalg.norm(D, axis=1))
        assert err.max() <= T_RAY, f"{label}: r = 0 crossing off by {err.max():.3g} of M / |D|"


def test_needle_rotations_agree():
    """the face of a needle is taken at the corner opposite its longest edge, so the rotations of one triangle give the same contact
    times within rounding (the example of a triangle 100 long and 0.05 wide, swept head-on at barycentrics (0.4, 0.4) and (0.2, 0.4))"""
    tri = np.array([[0, 0, 0], [100, -0.025, 0], [100, 0.025, 0]], np.float32)
    for r in (0.0, 0.01, 0.02):
        ts = []
        for k in range(3):
            V = np.roll(tri, -k, axis=0)
            q = so.queries(np.array([[80, 0, 1], [60, 0.005, -3]], np.float32), np.array([[0, 0, -1], [0, 0, 1]], np.float32), r, 5.0)
            hit, t, u, v = so.triangles(q, V[None, 0].repeat(2, 0), (V[1] - V[0])[None].repeat(2, 0), (V[2] - V[0])[None].repeat(2, 0))
            assert hit.all(), (r, k)
            ts.append(t)
        assert np.allclose(ts[0], ts[1], atol=1e-5) and np.allclose(ts[0], ts[2], atol=1e-5), (r, ts)
        assert np.allclose(ts[0], [1 - r, 3 - r], atol=1e-5)


def test_analytic_contacts():
    A = np.array([[0, 0, 0]], np.float32)
    e1, e2 = np.array([[4, 0, 0]], np.float32), np.array([[0, 4, 0]], np.float32)
    cases = [  # (c, r, D, tmax) -> (t, u, v)
        ((1, 1, 5), 1, (0, 0, -1), 10, (4, 0.25, 0.25)),        # head-on face, from above
        ((1, 1, -5), 1, (0, 0, 0.5), 20, (8, 0.25, 0.25)),      # from below (two-sided), D a half-unit
        ((2, -5, 0), 1, (0, 1, 0), 10, (4, 0.5, 0)),            # edge AB first, in the plane
        ((-5, 2, 0.5), 0.5, (1, 0, 0), 10, (5, 0, 0.5)),        # edge AC first, grazing the plane at height r
        ((3, 3, 0), 1, (1, 1, 0), 10, None),                     # edge BC first: moving away from it - no contact
        ((1, 1, 0.5), 1, (0, 0, 1), 10, "overlap"),              # initial overlap
    ]
    for c, r, D, tmax, want in cases:
        q = so.queries(np.array([c], np.float32), np.array([D], np.float32), r, tmax)
        hit, t, u, v = so.triangles(q, A, e1, e2)
        if want is None:
            assert not hit[0], (c, D)
        elif want == "overlap":
            d2, cu, cv = co.triangles(q[:, :3], A, e1, e2)
            assert hit[0] and t[0] == 0 and u[0] == cu[0] and v[0] == cv[0]
        else:
            assert hit[0] and (t[0], u[0], v[0]) == want, (c, D, t, u, v)
    # edge BC from outside: the centre moves toward the hypotenuse x + y = 4 from (5, 5, 0) along -(1, 1, 0)
    q = so.queries(np.array([[5, 5, 0]], np.float32), np.array([[-1, -1, 0]], np.float32), 1, 10)
    hit, t, u, v = so.triangles(q, A, e1, e2)
    assert hit[0] and abs(t[0] - (3 - 1 / np.sqrt(2))) < 1e-6 and abs(u[0] - 0.5) < 1e-6 and abs(v[0] - 0.5) < 1e-6
    # vertex A first: approaching along the diagonal from below-left, no edge parameter in [0, 1] at contact
    q = so.queries(np.array([[-3, -3, 0]], np.float32), np.array([[1, 1, 0]], np.float32), 1, 10)
    hit, t, u, v = so.triangles(q, A, e1, e2)
    assert hit[0] and abs(t[0] - (3 - 1 / np.sqrt(2))) < 1e-6 and (u[0], v[0]) == (0, 0)
    # vertex B first, from beyond it along the x axis's continuation but off the plane
    q = so.queries(np.array([[9, 0, 0.6]], np.float32), np.array([[-1, 0, 0]], np.float32), 1, 10)
    hit, t, u, v = so.triangles(q, A, e1, e2)
    assert hit[0] and abs(t[0] - 4.2) < 1e-6 and (u[0], v[0]) == (1, 0)
    # past tmax: no contact; exactly at tmax: contact
    q = so.queries(np.array([[1, 1, 5]] * 2, np.float32), np.array([[0, 0, -1]] * 2, np.float32), 1, np.array([3.5, 4], np.float32))
    hit, t, _, _ = so.triangles(q, np.repeat(A, 2, 0), np.repeat(e1, 2, 0), np.repeat(e2, 2, 0))
    assert hit.tolist() == [False, True] and t[1] == 4


def test_zero_radius_matches_ray_crossing():
    """r = 0 is a ray: on robust crossings (barycentrics >= 1e-5, t away from 0 and tmax) t is the fp64 crossing within T_RAY M / |D|"""
    rng = np.random.default_rng(8)
    n = 6000
    A = (rng.normal(size=(n, 3)) * 3).astype(np.float32)
    e1, e2 = rng.normal(size=(n, 3)).astype(np.float32), rng.normal(size=(n, 3)).astype(np.float32)
    start = A + rng.normal(size=(n, 3)).astype(np.float32) * 4
    target = A + rng.uniform(0, 0.5, (n, 1)) * e1 + rng.uniform(0, 0.5, (n, 1)) * e2 + rng.normal(size=(n, 3)) * 0.3
    D = (target - start).astype(np.float32)
    q = so.queries(start, D, 0.0, 2.0)
    hit, t, u, v = so.triangles(q, A, e1, e2)
    tri = np.stack([A, A + e1.astype(np.float64), A + e2.astype(np.float64)], 1)
    t64 = np.empty(n)
    b = np.empty((n, 3))
    for i in range(0, n, 500):
        s = slice(i, i + 500)
        tt, uu, vv, _ = solve64(start[s], D[s], tri[s])
        idx = np.arange(tt.shape[0])
        t64[s], b[s] = tt[idx, idx], np.stack([1 - uu[idx, idx] - vv[idx, idx], uu[idx, idx], vv[idx, idx]], 1)
    M = magnitude(q, A.astype(np.float64), e1.astype(np.float64), e2.astype(np.float64))
    tb = T_RAY * M / np.linalg.norm(D.astype(np.float64), axis=1)
    robust = (b >= 1e-5).all(1) & (t64 > tb) & (t64 < 2.0 - tb)
    assert robust.sum() > 1000
    assert hit[robust].all(), "a robust crossing missed"
    assert (np.abs(t[robust] - t64[robust]) <= tb[robust]).all(), np.max(np.abs(t[robust] - t64[robust]) / tb[robust])
    check_fp64(q, A, e1, e2, "r = 0")


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def scene_queries(v, rng, n=1500, short=True):
    """sweeps over a scene: short ones from near the surface in random directions (tmax 5 % of the extent, unit D), long ones from
    outside the box across it (D the displacement, tmax 1), radii 0, 0.1 % and 1 % of the extent and a few invalid queries"""
    tri = v.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    lo, hi = tri.reshape(-1, 3).min(0), tri.reshape(-1, 3).max(0)
    ext = float((hi - lo).max())
    k = rng.integers(0, tri.shape[0], n)
    w = rng.dirichlet((1, 1, 1), n)
    near = (w[:, :, None] * tri[k]).sum(1) + rng.normal(size=(n, 3)) * 0.01 * ext
    mid = (lo + hi) / 2
    far = mid + unit(rng.normal(size=(n, 3))) * ext
    to = mid + rng.uniform(-0.5, 0.5, (n, 3)) * (hi - lo)
    r = np.choose(rng.integers(0, 3, n), [np.zeros(n), np.full(n, 1e-3 * ext), np.full(n, 1e-2 * ext)])
    qs = so.queries(near, unit(rng.normal(size=(n, 3))), r, 0.05 * ext)
    ql = so.queries(far, to - far, r, 1.0)
    q = np.concatenate([qs, ql])
    q[0, 0], q[1, 3], q[2, 7], q[3, 5], q[4, 3], q[5, 7] = np.nan, -1, np.nan, np.inf, np.inf, np.inf
    return q


def check_same(nodes, idx, v, q, label):
    b = so.brute(nodes, idx, v, q)
    w = so.walk(nodes, idx, v, q)
    assert np.array_equal(bits(b), bits(w)), f"{label}: pruned walk differs from the brute force"
    bb = so.brute(nodes, idx, v, q, any_=True)
    assert np.array_equal(so.walk(nodes, idx, v, q, any_=True), bb), f"{label}: blocked bits of the walk differ"
    found = so.record_prims(b) != so.NO_PRIM
    got = np.unpackbits(bb.view(np.uint8), bitorder="little")[: q.shape[0]].astype(bool)
    assert np.array_equal(got, found), f"{label}: blocked bit is not 'sphere_cast finds a contact'"
    miss = ~found
    assert np.array_equal(bits(b[miss, 0]), bits(q[miss, 7])) and (b[miss, 1:3] == 0).all(), f"{label}: miss records carry tmax"
    return b


@pytest.mark.parametrize("ntris", [1, 7, 2000])
def test_brute_force_equals_pruned_walk(ntris):
    v = scenes.procedural_scene(ntris, 11 + ntris)
    q = scene_queries(v, np.random.default_rng(ntris), n=500)
    for label, nodes, idx in builder_trees(v):
        b = check_same(nodes, idx, v, q, f"{label}-{ntris}")
        assert not (so.record_prims(b[:5]) != so.NO_PRIM).any(), "invalid queries get the miss record"
        if ntris == 2000:
            assert 0.05 < (so.record_prims(b) != so.NO_PRIM).mean() < 0.95


def test_failed_split_sbvh_brute_force_equals_pruned_walk():
    from tests.test_build_hq_shapes import fail_scene, fail_scene_hq
    v = fail_scene("snapped3k_q4")
    nodes, idx = fail_scene_hq("snapped3k_q4")[:2]
    check_same(nodes, idx, v, scene_queries(v, np.random.default_rng(6), n=400), "snapped3k_q4")


@pytest.mark.parametrize("fam", util.FAMILIES + ["shrunk", "dag"])
def test_families_brute_force_equals_pruned_walk(fam):
    v = scenes.procedural_scene(3000, 71)
    src = util.source_tree(v, "BuildHQ" if fam in ("A1", "DB") else "Build")
    nodes, idx = family(src, fam)
    check_same(nodes, idx, v, scene_queries(v, np.random.default_rng(9), n=400), fam)


def test_deep_and_one_leaf_trees():
    from tests.test_closest_point_gpu import chain_tree
    v = scenes.procedural_scene(400, 12)
    for m in (100, 255):
        nodes, idx = chain_tree(v, m)
        check_same(nodes, idx, v[: 3 * m], scene_queries(v[: 3 * m], np.random.default_rng(m), n=300), f"chain-{m}")
    w = scenes.procedural_scene(40, 4)
    one = np.zeros(2, co.portpy.NODE32)
    tri = w.reshape(-1, 4)[:, :3]
    one[0] = (tri.min(0), 0, tri.max(0), 40)
    check_same(one, np.arange(40, dtype=np.uint32), w, scene_queries(w, np.random.default_rng(4), n=300), "one leaf")


def scaled_tree(nodes, k):
    out = nodes.copy()
    out["aabbMin"] *= np.float32(2.0 ** k)
    out["aabbMax"] *= np.float32(2.0 ** k)
    return out


@pytest.mark.parametrize("k", [-40, -17, -1, 9, 40])
def test_power_of_two_scaling(k):
    """mesh, tree boxes, c, r and D times 2^k: the same records bit for bit (t is a time: unchanged)"""
    v = scenes.procedural_scene(2000, 5)
    nodes, idx = util.source_tree(v, "Build")[:2]
    q = scene_queries(v, np.random.default_rng(2), n=400)[6:]
    want = so.brute(nodes, idx, v, q)
    f = np.float32(2.0 ** k)
    vs, qs = v.copy(), q.copy()
    vs[:, :3] *= f
    qs[:, :7] *= f
    got = so.brute(scaled_tree(nodes, k), idx, vs, qs)
    assert np.array_equal(bits(got), bits(want)), f"2^{k}: {int((bits(got) != bits(want)).any(1).sum())} records differ"
    for A, e1, e2, qq, label in sweep_cases(n=500):
        if label.endswith("random") or label.endswith("grazing"):
            h0, t0, u0, v0 = so.triangles(qq, A, e1, e2)
            q2 = qq.copy()
            q2[:, :7] *= f
            h1, t1, u1, v1 = so.triangles(q2, A * f, e1 * f, e2 * f)
            assert np.array_equal(h0, h1) and np.array_equal(bits(t0), bits(t1)) and np.array_equal(bits(u0), bits(u1)) and np.array_equal(bits(v0), bits(v1)), label


@pytest.mark.parametrize("m", [-30, -3, 5, 30])
def test_direction_scaling(m):
    """D times 2^m and tmax times 2^-m: t times 2^-m, the same u, v and prim"""
    v = scenes.procedural_scene(2000, 6)
    nodes, idx = util.source_tree(v, "BuildHQ")[:2]
    q = scene_queries(v, np.random.default_rng(3), n=400)[6:]
    want = so.brute(nodes, idx, v, q)
    q2 = q.copy()
    q2[:, 4:7] *= np.float32(2.0 ** m)
    q2[:, 7] *= np.float32(2.0 ** -m)
    got = so.brute(nodes, idx, v, q2)
    assert np.array_equal(bits(got[:, 1:]), bits(want[:, 1:]))
    assert np.array_equal(bits(got[:, 0]), bits(want[:, 0] * np.float32(2.0 ** -m)))


@pytest.mark.parametrize("mode", ["random", "order"])
def test_signed_zero_twins(mode):
    """a mesh whose zeros are -0, and queries whose zero components are -0, give the +0 twin's records up to the sign of a zero"""
    v = util.signed_zero(scenes.procedural_scene(2000, 7), "pos")
    q = scene_queries(v, np.random.default_rng(4), n=400)[6:]
    q[::3, 4] = 0
    q[1::3, 5:7] = 0
    nodes, idx = util.source_tree(v, "Build")[:2]
    want = so.brute(nodes, idx, v, q)
    vz = util.signed_zero(scenes.procedural_scene(2000, 7), mode)
    assert util.count_neg_zero(vz) > 0
    qz = q.copy()
    qz[qz == 0] = -0.0
    nz = nodes.copy()
    for f in ("aabbMin", "aabbMax"):
        nz[f][nz[f] == 0] = -0.0
    got = so.brute(nz, idx, vz, qz)
    plus = lambda a: bits(np.asarray(a, np.float32) + np.float32(0))
    assert np.array_equal(plus(got[:, :3]), plus(want[:, :3])) and np.array_equal(bits(got[:, 3]), bits(want[:, 3]))


def test_translated_scene_fp64():
    """a scene translated by 2^20: each triangle's contact is held to fp64 with M taken from the absolute coordinates"""
    for A, e1, e2, q, label in sweep_cases(seed=9, n=1500):
        if not label.startswith("random/"):
            continue
        T = np.float32(2.0 ** 20)
        A2 = (A + T).astype(np.float32)
        q2 = q.copy()
        q2[:, :3] += T
        M = np.max(np.abs(np.concatenate([q2[:, :3], A2, A2 + e1, A2 + e2, q2[:, :3] + q2[:, 7:8] * q2[:, 4:7]], 1)), 1).astype(np.float64)
        check_fp64(q2, A2, e1, e2, "translated/" + label, M=M)


def test_axis_aligned_sweeps():
    """sweeps with +-0 direction components in all 8 octants: fp64 rules per triangle, the walk on trees, and the -0 / +0 twins agree"""
    v = scenes.procedural_scene(2000, 19)
    nodes, idx = util.source_tree(v, "Build")[:2]
    rng = np.random.default_rng(5)
    tri = v.reshape(-1, 3, 4)[:, :, :3]
    lo, hi = tri.reshape(-1, 3).min(0), tri.reshape(-1, 3).max(0)
    n = 400
    qs = []
    for octant in range(8):
        sgn = np.array([1 if octant & (4 >> a) else -1 for a in range(3)], np.float32)
        for axis in range(3):
            c = lo + rng.uniform(0, 1, (n, 3)) * (hi - lo)
            D = np.zeros((n, 3), np.float32)
            D[:, axis] = sgn[axis]
            D[D == 0] = np.where(np.broadcast_to(sgn, (n, 3)) < 0, -0.0, 0.0)[D == 0]
            qs.append(so.queries(c, D, rng.uniform(0, 0.02, n) * (hi - lo).max(), (hi - lo).max()))
    q = np.concatenate(qs)
    b = check_same(nodes, idx, v, q, "axis-aligned")
    found = so.record_prims(b) != so.NO_PRIM
    assert found.mean() > 0.05
    q2 = q.copy()
    q2[:, 4:7] = np.where(q2[:, 4:7] == 0, np.float32(0), q2[:, 4:7])
    assert np.array_equal(bits(so.brute(nodes, idx, v, q2)), bits(b)), "-0 and +0 direction components differ"
    # per triangle against fp64, each query with its reported triangle (or a random one)
    prim = np.where(found, so.record_prims(b), rng.integers(0, tri.shape[0], q.shape[0]))
    A = tri[prim, 0].astype(np.float32)
    check_fp64(q, A, (tri[prim, 1] - A).astype(np.float32), (tri[prim, 2] - A).astype(np.float32), "axis-aligned")


def test_zero_length_sweeps_are_sphere_overlaps():
    """D = 0: the queries with a t = 0 record are those whose sphere overlaps the mesh (tbvh_sphere_overlap's bits), except within
    rounding of touching"""
    v = scenes.procedural_scene(3000, 23)
    nodes, idx = util.source_tree(v, "Build")[:2]
    q = scene_queries(v, np.random.default_rng(7), n=1500)[6:]
    q[:, 4:7] = 0
    b = so.brute(nodes, idx, v, q)
    cast = (so.record_prims(b) != so.NO_PRIM) & (b[:, 0] == 0)
    assert np.array_equal(cast, so.record_prims(b) != so.NO_PRIM), "a zero-length sweep touches at t = 0 or not at all"
    ob = co.brute(nodes, idx, v, q[:, :4], any_=True)
    over = np.unpackbits(ob.view(np.uint8), bitorder="little")[: q.shape[0]].astype(bool)
    diff = np.nonzero(cast != over)[0]
    assert cast.sum() > 100
    tri = v.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    for i in diff:   # only spheres that touch within rounding may differ
        d = fp64_closest(np.repeat(q[i: i + 1, :3], tri.shape[0], 0), tri[:, 0], tri[:, 1], tri[:, 2]).min()
        assert abs(d - q[i, 3]) <= 1e-6 * max(np.abs(tri).max(), 1), (i, d, q[i, 3])


def test_python_query_rows():
    """the Python rows: (n, 3) + radii / tmax, (n, 4) rows, (n, 8) records; mismatched shapes raise before any native call"""
    rng = np.random.default_rng(1)
    c, d = rng.normal(size=(5, 3)).astype(np.float32), rng.normal(size=(5, 3)).astype(np.float32)
    q = api._np_sweeps(c, d, 0.5, None)
    assert q.shape == (5, 8) and (q[:, 3] == 0.5).all() and np.isinf(q[:, 7]).all() and np.array_equal(q[:, 4:7], d)
    q4 = api._np_sweeps(q[:, :4], q[:, 4:8], None, None)
    assert np.array_equal(bits(q4), bits(q))
    assert np.array_equal(bits(api._np_sweeps(q, None, None, None)), bits(q))
    r = np.arange(5, dtype=np.float32)
    assert np.array_equal(api._np_sweeps(c, d, r, r)[:, [3, 7]], np.stack([r, r], 1))
    for args in ((c, None, 1, None), (c, d, None, None), (q[:, :4], d, 1, None), (c, q[:, 4:8], 1, 2.0), (c, d[:4], 1, None),
                 (c, d, np.ones(4), None), (c, d, 1, np.ones(6)), (q, d, None, None), (q[:, :5], None, None, None)):
        with pytest.raises(api.TbvhError):
            api._np_sweeps(*args)
