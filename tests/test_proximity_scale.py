"""The proximity queries away from the unit scale, on the host restatements (tests/closest_oracle.c, sdf_oracle.c, wn_oracle.c;
DESIGN.md §4.9-4.11), without a GPU.  Multiplying a mesh and its queries by 2^k is exact, so inside the window W = [-40, 40] every
result must follow it exactly: closest-point and signed distances scale by 2^k, and weights, prims, signs, sphere bits, signed-distance
tables and winding numbers keep their bits.  That needs no reference and catches any over- or underflow.  Independently, at every k the
results are held to fp64 at the bounds the unit-scale suites measured, scaled by 2^k; translated meshes are held to fp64 on their exact
fp32 inputs; a mesh whose zeros are -0 gives its +0 twin's bits; and outside W the documented limits are pinned."""
import numpy as np
import pytest

from tests import closest_oracle as co, sdf_oracle as so, util, wn_oracle as wo
from tests.test_closest_point import builder_trees, fp64_closest
from tests.test_signed_distance import cube, icosphere, soup, star, torus, winding
from tests.test_winding_number import BETA_BOUND, EXACT_BOUND, hemisphere, two_spheres

W = list(range(-40, 41))
# The expansion's records hold the second moments M, of degree 3 in lengths; for these meshes (extent about 2) the leaf records' M
# become subnormal below 2^-34, so finite-beta winding numbers keep their bits from 2^-34 up and only their fp64 bounds below (DESIGN 4.11)
WN_LOW = -34
OUTSIDE = [-126, -100, -60, 60, 90]                  # the rest of the SCALE family of tests/test_offatrium_gpu.py
SHIFT = [1048576.0, -12582912.0]                     # +2^20, -3 * 2^22, as tests/test_offatrium_gpu.py
ZERO = ["neg", "random", "order"]                     # against the "pos" twin (util.signed_zero)
BETAS = [1.5, 2.0, 4.0, np.inf]
CP_BOUND = 2e-6                                       # closest point: of the magnitude (DESIGN 4.9 item 1)

CLOSED = {"icosphere": lambda: icosphere(2), "torus": lambda: torus(nu=16, nv=8), "star": star, "cube": cube}
OPEN = {"hemisphere": hemisphere, "two_spheres": two_spheres}
MESHES = dict(CLOSED, **OPEN)


def queries(V, F, seed, n=240):
    """uniform in 1.3 times the box, jittered surface points, far points; r (for the sphere bits and r_max) of mixed sizes, some inf"""
    rng = np.random.default_rng(seed)
    V = np.asarray(V, np.float64)
    lo, hi = V.min(0), V.max(0)
    c, half, ext = (lo + hi) / 2, (hi - lo) / 2 * 1.3 + 1e-3, (hi - lo).max()
    tri = V[F]
    k = rng.integers(0, F.shape[0], n)
    w = rng.dirichlet((1, 1, 1), n)
    P = np.concatenate([c + rng.uniform(-1, 1, (n, 3)) * half, (tri[k] * w[:, :, None]).sum(1) + rng.normal(size=(n, 3)) * 0.03 * ext,
                        c + rng.normal(size=(n // 8, 3)) * 20 * ext])
    q = np.zeros((P.shape[0], 4), np.float32)
    q[:, :3] = P
    q[:, 3] = np.where(rng.random(P.shape[0]) < 0.25, np.inf, rng.uniform(0, 0.3 * ext, P.shape[0]))
    return q


def scaled_q(q, k):
    """queries (and their radii) times exactly 2^k"""
    q = q.copy()
    q[:, :4] = np.ldexp(q[:, :4], k)
    return q


_BASE = {}


def base(name):
    """(V, F, soup, queries) of a mesh at unit scale"""
    if name not in _BASE:
        V, F = MESHES[name]()
        _BASE[name] = (V, F, soup(V, F), queries(V, F, len(name)))
    return _BASE[name]


def results(v, q, name):
    """every restated result of one mesh: closest records (Build tree), sphere words, signed-distance table and records (closed meshes),
    winding numbers at every beta (the Build tree)"""
    _, nodes, idx = builder_trees(v)[0]
    out = {"cp": co.walk(nodes, idx, v, q), "overlap": co.walk(nodes, idx, v, q, any_=True)}
    qi = q.copy()
    qi[:, 3] = np.inf
    out["cp_inf"] = co.walk(nodes, idx, v, qi)
    if name in CLOSED:
        table = so.prepare(v)
        out["sd_table"] = table
        out["sd"] = so.brute(nodes, idx, v, qi, table, walk=True)
    t = wo.Table(nodes, idx, v)
    assert t.flag == 0
    for b in BETAS:
        out[f"wn{b}"] = t.query(q, b)
    return out


_AT = {}


def at(name, k):
    if (name, k) not in _AT:
        V, F, v, q = base(name)
        _AT[(name, k)] = results(util.scaled(v, k), scaled_q(q, k), name)
    return _AT[(name, k)]


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def diff(a, b):
    return int((bits(a) != bits(b)).sum())


def scale_records(rec, k):
    """a {d, u, v, prim} record array with d times 2^k"""
    r = np.array(rec, np.float32)
    r[:, 0] = np.ldexp(r[:, 0], k)
    return r


# ---- power-of-two covariance ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(MESHES))
def test_power_of_two_covariance(name):
    """for every k in W: closest-point and signed distances are the k = 0 ones times 2^k with identical u, v, prim (and sign); sphere
    words, signed-distance tables and exact winding numbers have identical bits, and so do winding numbers at beta 1.5, 2 and 4 from
    WN_LOW up"""
    r0 = at(name, 0)
    bad = []
    for k in W:
        rk = results(util.scaled(base(name)[2], k), scaled_q(base(name)[3], k), name)
        for key, want in r0.items():
            if key in ("cp", "cp_inf", "sd"):
                want = scale_records(want, k)
            if key in ("wn1.5", "wn2.0", "wn4.0") and k < WN_LOW:
                continue
            n = diff(rk[key], want)
            if n:
                bad.append(f"k={k} {key}: {n} words")
    assert not bad, f"{name}: " + "; ".join(bad[:12])


# ---- fp64 anchors --------------------------------------------------------------------------------------------------------------
def fp64_nearest(v, P):
    """the fp64 distance from each point to the soup v (float32 inputs, exactly)"""
    tri = np.asarray(v, np.float64).reshape(-1, 3, 4)[:, :, :3]
    P = np.asarray(P, np.float64)[:, :3]
    n, m = P.shape[0], tri.shape[0]
    pp = np.repeat(P, m, 0)
    d = fp64_closest(pp, np.tile(tri[:, 0], (n, 1)), np.tile(tri[:, 1], (n, 1)), np.tile(tri[:, 2], (n, 1)))
    return d.reshape(n, m).min(1)


_FP64 = {}


def fp64(name):
    """fp64 nearest distance and winding number of the unit-scale inputs; power-of-two scaling is exact in fp64 as well, so the
    references at 2^k are these times 2^k (distances) and these (winding numbers)"""
    if name not in _FP64:
        V, F, v, q = base(name)
        tri = np.asarray(v, np.float64).reshape(-1, 3, 4)[:, :, :3]
        Vx = tri.reshape(-1, 3)
        Fx = np.arange(Vx.shape[0]).reshape(-1, 3)
        d64 = fp64_nearest(v, q)
        w64 = winding(Vx, Fx, q[:, :3].astype(np.float64))
        mag = np.maximum(np.abs(q[:, :3]).max(1), np.abs(tri).max())
        ext = np.ptp(Vx, 0).max()
        _FP64[name] = (d64, w64, mag, ext)
    return _FP64[name]


def check_fp64(name, r, k, d64, w64, mag, ext, q):
    """r: the results at 2^k; d64, mag, ext already at 2^k; q at 2^k"""
    fails = []
    d = r["cp_inf"][:, 0].astype(np.float64)
    tol = CP_BOUND * mag
    if not (np.abs(d - d64) <= tol).all():
        fails.append(f"closest point off by {(np.abs(d - d64) / tol).max():.3g} x its bound")
    # sphere bits agree with fp64 wherever |d64 - r| is above the closest-point bound
    rr = q[:, 3].astype(np.float64)
    want = d64 <= rr
    got = (np.unpackbits(bits(r["overlap"]).view(np.uint8), bitorder="little")[: q.shape[0]]).astype(bool)
    clear = np.abs(d64 - rr) > tol
    if (got != want)[clear].any():
        fails.append(f"{int((got != want)[clear].sum())} sphere bits differ from fp64")
    away = d64 > 1e-3 * ext
    if "sd" in r:
        inside = w64 > 0.5
        neg = r["sd"][:, 0] < 0
        if (neg != inside)[away].any():
            fails.append(f"{int((neg != inside)[away].sum())} signed-distance signs wrong")
    for b, bound in ((np.inf, EXACT_BOUND), (2.0, BETA_BOUND[2.0]), (4.0, BETA_BOUND[4.0])):
        e = np.abs(r[f"wn{b}"].astype(np.float64) - w64)[away]
        if not (e <= bound).all():
            fails.append(f"winding number at beta {b} off by {np.nanmax(np.where(np.isnan(e), np.inf, e)):.3g} (bound {bound})")
    return fails


@pytest.mark.parametrize("name", list(MESHES))
def test_fp64_anchors_at_every_scale(name):
    """at every k in W: closest point within 2e-6 of the magnitude, sphere bits where the fp64 distance is clear of r, exact signs on the
    closed meshes and winding numbers within 3e-6 exact, 0.11 at beta 2, 0.017 at beta 4, at queries farther than 1e-3 of the extent"""
    d64, w64, mag, ext = fp64(name)
    q0 = base(name)[3]
    bad = []
    for k in W:
        q = scaled_q(q0, k)
        r = results(util.scaled(base(name)[2], k), q, name)
        f = check_fp64(name, r, k, np.ldexp(d64, k), w64, np.ldexp(mag, k), np.ldexp(ext, k), q)
        bad += [f"k={k}: {x}" for x in f]
    assert not bad, f"{name}: " + "; ".join(bad[:12])


# ---- translated and signed-zero families ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("shift", SHIFT)
@pytest.mark.parametrize("name", ["icosphere", "torus", "hemisphere", "two_spheres"])
def test_translated_against_fp64(name, shift):
    """meshes and queries moved by millions of units: fp64 runs on the exact fp32 inputs, closest-point tolerances scale with the
    coordinates' magnitude; signs and winding numbers at the unit-scale bounds"""
    V, F, v0, q0 = base(name)
    v = util.translated(v0, shift)
    q = q0.copy()
    q[:, :3] = q[:, :3] + np.float32(shift)
    r = results(v, q, name)
    tri = np.asarray(v, np.float64).reshape(-1, 3, 4)[:, :, :3]
    Vx = tri.reshape(-1, 3)
    d64 = fp64_nearest(v, q)
    w64 = winding(Vx, np.arange(Vx.shape[0]).reshape(-1, 3), q[:, :3].astype(np.float64))
    mag = np.maximum(np.abs(q[:, :3]).max(1), np.abs(tri).max())
    bad = check_fp64(name, r, 0, d64, w64, mag, np.ptp(Vx, 0).max(), q)
    assert not bad, f"{name} + {shift}: " + "; ".join(bad)


@pytest.mark.parametrize("mode", ZERO)
@pytest.mark.parametrize("name", ["icosphere", "cube", "hemisphere"])
def test_signed_zero_twin(name, mode):
    """zeros snapped to -0 (every one, a seeded sign each, or every order in a triangle) give the bits of the +0 twin: records, sphere
    words, signed-distance tables and records, winding numbers; queries with +-0 coordinates included"""
    V, F, v0, q0 = base(name)
    v = util.signed_zero(v0, mode, seed=3, frac=0.2)
    vp = util.signed_zero(v0, "pos", seed=3, frac=0.2)
    assert util.count_neg_zero(v) > 0
    q = np.concatenate([q0, vp[:40]])
    q[-40:, 3] = np.inf
    qn = util.signed_zero(q, mode, seed=5, frac=0.2)
    qp = util.signed_zero(q, "pos", seed=5, frac=0.2)
    a, b = results(v, qn, name), results(vp, qp, name)
    # the one place a sign of zero survives: a face normal component that is exactly 0 is -0 or +0 as e1 x e2 rounds it (DESIGN 4.10);
    # it enters the sign only through ( p - c ) . N, where a zero product cannot make a nonzero sum negative
    assert "sd_table" not in a or np.array_equal(a["sd_table"], b["sd_table"]), "signed-distance tables differ in value"
    bad = [f"{key}: {diff(a[key], b[key])} words" for key in a if key != "sd_table" and diff(a[key], b[key])]
    assert not bad, f"{name} {mode}: " + "; ".join(bad)


# ---- outside the window --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", OUTSIDE)
def test_outside_the_window(k):
    """What DESIGN 4.9-4.11 state beyond W, pinned on the icosphere against fp64 on the exact fp32 inputs:
    * the exact winding number (beta = inf) keeps its 3e-6 bound at every scale of the family: its terms are scaled per triangle;
    * at 2^-60 closest-point distances are within 2e-6 of the magnitude plus 2^-72 (a squared distance there is subnormal), every
      signed-distance sign is exact and the expansion keeps its beta 2 and 4 bounds;
    * at 2^60 and above the expansion's records overflow: a finite-beta winding number may be NaN, never a wrong finite number that
      is off by more than its bound;
    * sphere bits are exactly "closest point with r_max = r finds a triangle" at every scale (§4.9 item 5)."""
    V, F, v0, q0 = base("icosphere")
    v, q = util.scaled(v0, k), scaled_q(q0, k)
    r = results(v, q, "icosphere")
    tri = np.asarray(v, np.float64).reshape(-1, 3, 4)[:, :, :3]
    Vx = tri.reshape(-1, 3)
    w64 = winding(Vx, np.arange(Vx.shape[0]).reshape(-1, 3), q[:, :3].astype(np.float64))
    d64 = fp64_nearest(v, q)
    away = d64 > 1e-3 * np.ptp(Vx, 0).max()
    assert (np.abs(r["wninf"].astype(np.float64) - w64)[away] <= EXACT_BOUND).all()
    found = bits(r["cp"])[:, 3] != co.NO_PRIM
    got = np.unpackbits(bits(r["overlap"]).view(np.uint8), bitorder="little")[: q.shape[0]].astype(bool)
    assert np.array_equal(got, found)
    for b in (2.0, 4.0):
        e = np.abs(r[f"wn{b}"].astype(np.float64) - w64)[away]
        assert (np.isnan(e) | (e <= BETA_BOUND[b])).all(), f"beta {b}"
        if k < 60:
            assert not np.isnan(e).any(), f"beta {b}"
    if k == -60:
        mag = np.maximum(np.abs(q[:, :3]).max(1), np.abs(tri).max())
        assert (np.abs(r["cp_inf"][:, 0] - d64) <= CP_BOUND * mag + 2.0 ** -72).all()
        assert ((r["sd"][:, 0] < 0) == (w64 > 0.5))[away].all()
