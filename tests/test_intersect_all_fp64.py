"""The multi-hit ray query (DESIGN.md §4.14) against fp64, on the host restatement (tests/allhits_oracle.c), without a GPU.  The other
suites hold the restatement's brute force and walk to each other and the device to both; this file checks which triangles a ray reports
and their t against an independent reference: a plain fp64 solve of O + t D = v0 + u e1 + v e2 on the exact fp32 corners, with O and D
the record's own (the stored, normalised direction).  For every ray with count <= k (k = 64):
* every robust crossing is among the records: all three barycentrics >= 1e-5, the crossing point farther than 4 ulps of the largest
  coordinate magnitude (ray origin and corners) from each edge of the triangle, and t clear of 0 and tmax by the t bound;
* no record is a robust miss (a barycentric <= -1e-5 with the point as far outside, or t outside [0, tmax] by more than the bound);
* |t - t64| <= 1e-6 |O - v0| / |D| on every record, and the records are in t order to within that bound;
* robust <= count <= robust + ambiguous.
That holds over every builder's tree (the failed-split SBVH included), at 2^k across the window WINDOW, translated by 3e5 and 3e6 with
rays near the geometry, and on signed-zero twins, which also give their +0 twin's prims and counts with t, u and v equal as values.
Below the window mt_test's absolute determinant threshold (|e1 . (D x e2)| < 1e-6, as BVH::Intersect) drops crossings; the test pins
where that begins.  Through a TLAS the same rules hold for affine instances, with the BLAS corners moved to world space in fp64 (t is
shared between world and BLAS space, §4.3d); projective instances are out of scope here: their world-space triangles are not planar
images under a division-free map, so a world-space fp64 solve is not their definition."""
import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import rays as R, scenes
from tests import allhits_oracle as ao, util
from tests.test_closest_point import builder_trees

K = 64
T_BOUND = 1e-6          # of |O - v0| / |D|
BARY = 1e-5
ULPS = 4                 # coordinate ulps a robust crossing keeps from each edge
EPS32 = 2.0 ** -23


def solve64(O, D, tri):
    """fp64 (t, u, v, det) of rays (n, 3) against triangles (m, 3, 3) -> (n, m) arrays"""
    O, D, tri = (np.asarray(x, np.float64) for x in (O, D, tri))
    v0, e1, e2 = tri[:, 0], tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    h = np.cross(D[:, None, :], e2[None])                     # (n, m, 3)
    det = np.einsum("mk,nmk->nm", e1, h)
    s = O[:, None, :] - v0[None]
    q = np.cross(s, e1[None])
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / det
        u = np.einsum("nmk,nmk->nm", s, h) * inv
        v = np.einsum("nk,nmk->nm", D, q) * inv
        t = np.einsum("mk,nmk->nm", e2, q) * inv
    return t, u, v, det


def classify(rays, tri, mag=None):
    """fp64 per (ray, triangle) of rays against triangles (m, 3, 3): t64, u, v, the robust-hit mask, the robust-miss mask and the t bound;
    mag: for a TLAS, the length of the ray transform's rounding: the t bound and the edge margin are taken from it over the cosine of the
    ray's angle to the normal where that is larger"""
    tri = np.asarray(tri, np.float64)
    O, D = rays["O"].astype(np.float64), rays["D"].astype(np.float64)
    tmax = rays["t"].astype(np.float64)
    t, u, w, det = solve64(O, D, tri)
    with np.errstate(invalid="ignore"):
        b = np.stack([1 - u - w, u, w], -1)                   # barycentrics of v0, v1, v2 (NaN where det == 0)
    # the coordinate ulp at the crossing: of the largest magnitude among the ray origin and the triangle's corners
    M = np.maximum(np.abs(O).max(1)[:, None], np.abs(tri).max((1, 2))[None])
    ulp = ULPS * EPS32 * M
    if mag is not None:
        # a ray moved by d across the plane moves its crossing by d / cos along it and its t by d / cos: the ray transform's rounding
        with np.errstate(divide="ignore", invalid="ignore"):
            cos = np.abs(det) / (np.linalg.norm(D, axis=1)[:, None] * np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)[None])
        mag = mag / cos
        ulp = ulp / cos
    # distance from P to each edge line: barycentric of the opposite corner times that corner's height over the edge
    e = [tri[:, 2] - tri[:, 1], tri[:, 0] - tri[:, 2], tri[:, 1] - tri[:, 0]]
    area2 = np.linalg.norm(np.cross(e[2], -e[1]), axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        height = [area2 / np.linalg.norm(x, axis=1) for x in e]
    with np.errstate(invalid="ignore"):
        edist = np.stack([b[..., c] * height[c][None] for c in range(3)], -1)
    L = np.linalg.norm(O[:, None, :] - tri[None, :, 0], axis=2)
    tb = T_BOUND * (L if mag is None else np.maximum(L, mag)) / np.linalg.norm(D, axis=1)[:, None]
    finite = np.isfinite(t) & (det != 0)
    inside = finite & (b >= BARY).all(-1) & (edist > ulp[..., None]).all(-1)
    hit = inside & (t > tb) & (t < tmax[:, None] - tb)
    out = finite & (((b <= -BARY) & (-edist > ulp[..., None])).any(-1) | (t < -tb) | (t > tmax[:, None] + tb))
    miss = out | ~finite
    return t, u, w, hit, miss, tb


def check_rules(rays, tri, hits, counts, k=K, p=None, mag=None):
    """the rules of the module docstring on one result; p: each record's triangle index into tri (default: its prim) -> {worst t error
    as a fraction of the bound, robust crossings missed, records that are robust misses, records out of order, counts outside the
    range, robust crossings, rays checked}; asserts nothing"""
    t64, u64, v64, hit, miss, tb = classify(rays, tri, mag)
    p = ao.prims(hits) if p is None else p
    worst, missed, wrong, order, outside, total = 0.0, 0, 0, 0, 0, 0
    ok = counts <= k
    for i in np.nonzero(ok)[0]:
        c = int(counts[i])
        js = p[i, :c].astype(np.int64)
        rec_t = hits[i, :c, 0].astype(np.float64)
        if c:
            err = np.abs(rec_t - t64[i, js]) / tb[i, js]
            worst = max(worst, float(np.nan_to_num(err, nan=np.inf).max()))
            bound = tb[i, js]
            order += int((rec_t[1:] < rec_t[:-1] - bound[1:] - bound[:-1]).sum())
            wrong += int(miss[i, js].sum())
        robust = np.nonzero(hit[i])[0]
        total += robust.shape[0]
        missed += int(np.setdiff1d(robust, js).shape[0])
        amb = int((~hit[i] & ~miss[i]).sum())
        outside += int(not (robust.shape[0] <= c <= robust.shape[0] + amb))
    return {"worst": worst, "missed": missed, "wrong": wrong, "order": order, "count": outside, "robust": total, "rays": int(ok.sum())}


def assert_rules(res, label):
    assert res["rays"] > 0 and res["robust"] > 0, label
    assert res["worst"] <= 1.0, f"{label}: t off by {res['worst']:.3g} x its bound"
    assert res["missed"] == 0, f"{label}: {res['missed']} robust crossings missing"
    assert res["wrong"] == 0, f"{label}: {res['wrong']} records are robust misses"
    assert res["order"] == 0, f"{label}: {res['order']} records out of t order"
    assert res["count"] == 0, f"{label}: {res['count']} counts outside [robust, robust + ambiguous]"


def inside_rays(v, n, seed, tmax=np.inf):
    """n rays from uniform points of the scene's box in random directions"""
    rng = np.random.default_rng(seed)
    lo, hi = (np.asarray(x, np.float64) for x in scenes.scene_bounds(v))
    O = (lo + rng.uniform(0, 1, (n, 3)) * (hi - lo)).astype(np.float32)
    return R.gpu_records(R.make_rays(O, rng.normal(size=(n, 3)).astype(np.float32), np.float32(tmax)))


def near_rays(v, n, seed):
    """n rays from points near the geometry (a jittered surface point, 0.5 to 3 units off) aimed back across it, tmax finite"""
    rng = np.random.default_rng(seed)
    tri = v.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    k = rng.integers(0, tri.shape[0], n)
    w = rng.dirichlet((1, 1, 1), n)
    p = (w[:, :, None] * tri[k]).sum(1)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    O = p - d * rng.uniform(0.5, 3.0, (n, 1))
    r = R.gpu_records(R.make_rays(O.astype(np.float32), d.astype(np.float32), np.float32(40.0)))
    return r


_SCENE = {}


def scene():
    if "v" not in _SCENE:
        _SCENE["v"] = scenes.procedural_scene(2000, 33)
        _SCENE["rays"] = inside_rays(_SCENE["v"], 300, 1)
    return _SCENE["v"], _SCENE["rays"]


def run(v, rays, nodes, idx, k=K):
    """the restatement's definition over (nodes, idx), and its rules against fp64 -> (rules, hits, counts)"""
    h, c, _ = ao.brute(nodes, idx, v, rays, k)
    return check_rules(rays, v.reshape(-1, 3, 4)[:, :, :3], h, c, k), h, c


# The window: 2^k from WINDOW_LOW to 2^20 for this scene and its rays.  mt_test's threshold |e1 . (D x e2)| < 1e-6 is absolute, and the
# determinant scales by 4^k with a unit D, so below the window it drops the crossings of the smallest and the most oblique triangles first
# (2^-10: 8 robust crossings lost), and at 2^-20 every one.
WINDOW_LOW = -9
WINDOW = list(range(WINDOW_LOW, 21))
SHIFT = [3e5, 3e6]
ZERO = ["neg", "random", "order"]


@pytest.mark.parametrize("builder", [0, 1, 2, 3])
def test_every_builder(builder):
    v, rays = scene()
    label, nodes, idx = builder_trees(v)[builder]
    res = run(v, rays, nodes, idx)[0]
    print(label, res)
    assert_rules(res, label)


def test_failed_split_sbvh():
    from tests.test_build_hq_shapes import fail_scene, fail_scene_hq
    v = fail_scene("snapped3k_q4")
    nodes, idx = fail_scene_hq("snapped3k_q4")[:2]
    assert_rules(run(v, inside_rays(v, 300, 3), nodes, idx)[0], "snapped3k_q4")


def test_power_of_two_window():
    """every k in WINDOW keeps the rules; the first k below it loses robust crossings, and 2^-20 loses them all"""
    v, rays = scene()
    worst = 0.0
    for k in WINDOW:
        vs = util.scaled(v, k)
        o = portpy.PortBVH(vs)
        res = run(vs, util.scaled_rays(rays, k), o.nodes, o.prim_idx)[0]
        assert_rules(res, f"2^{k}")
        worst = max(worst, res["worst"])
    print(f"worst t error {worst * T_BOUND:.3g} of |O - v0| / |D| over 2^{WINDOW_LOW} .. 2^20")
    for k in (WINDOW_LOW - 1, -20):
        vs = util.scaled(v, k)
        o = portpy.PortBVH(vs)
        res, h, c = run(vs, util.scaled_rays(rays, k), o.nodes, o.prim_idx)
        print(f"2^{k}: {res}")
        assert res["missed"] > 0, f"2^{k} loses no crossing: the window is wider than WINDOW_LOW states"
        if k == -20:
            assert res["missed"] == res["robust"] > 300 and (c == 0).all()


@pytest.mark.parametrize("shift", SHIFT)
def test_translated(shift):
    """the scene and rays near it (0.5 to 3 units off the surface) and from inside its box moved by 3e5 and 3e6, over Build and BuildHQ
    trees"""
    v, rays = scene()
    vt = util.translated(v, shift)
    near = near_rays(v, 300, 2)
    for r in (near, rays.copy()):
        r["O"] = r["O"] + np.float32(shift)
    for label, nodes, idx in (builder_trees(vt)[0], builder_trees(vt)[2]):
        for name, r in (("near", near), ("inside", rays)):
            ro = r.copy()
            ro["O"] = r["O"] + np.float32(shift) if name == "inside" else r["O"]
            res = run(vt, ro, nodes, idx)[0]
            print(f"+{shift} {label} {name}: {res}")
            assert_rules(res, f"+{shift} {label} {name}")


@pytest.mark.parametrize("mode", ZERO)
def test_signed_zero_twins(mode):
    """the rules on a scene whose snapped zeros are -0, and its +0 twin's prims and counts, with t, u and v equal as values"""
    v0, rays = scene()
    v, vp = util.signed_zero(v0, mode, seed=3, frac=0.2), util.signed_zero(v0, "pos", seed=3, frac=0.2)
    assert util.count_neg_zero(v) > 0
    for label, nodes, idx in builder_trees(v)[:3]:
        res, h, c = run(v, rays, nodes, idx)
        assert_rules(res, f"{mode} {label}")
    o, op = portpy.PortBVH(v), portpy.PortBVH(vp)
    h, c, _ = ao.brute(o.nodes, o.prim_idx, v, rays, K)
    hp, cp, _ = ao.brute(op.nodes, op.prim_idx, vp, rays, K)
    assert np.array_equal(c, cp) and np.array_equal(ao.prims(h), ao.prims(hp)), f"{mode}: prims or counts differ from the +0 twin"
    assert np.array_equal(h[..., :3], hp[..., :3]), f"{mode}: t, u or v differ in value from the +0 twin"


# ---- through a TLAS ----------------------------------------------------------------------------------------------------------------
def rotations(n, rng):
    q, r = np.linalg.qr(rng.normal(size=(n, 3, 3)))
    return q * np.sign(np.diagonal(r, axis1=1, axis2=2))[:, None, :]


def affine_families(seed=11):
    """name -> transforms (n, 16): rigid, non-uniform scale (a rotation times a diagonal of 0.5 to 2), every permutation and mirror,
    and rigid moved by 2^20"""
    from tests.test_tlas_update import update_families
    rng = np.random.default_rng(seed)

    def build(n, shift=0.0, scale=False):
        t = np.zeros((n, 4, 4), np.float32)
        m = rotations(n, rng)
        if scale:
            m = m * rng.uniform(0.5, 2.0, (n, 1, 3))
        t[:, :3, :3] = m
        t[:, :3, 3] = rng.uniform(-30, 30, (n, 3)) + shift
        t[:, 3, 3] = 1
        return t.reshape(-1, 16)
    return {"rigid": build(24), "nonuniform_scale": build(24, scale=True),
            "permutation_mirror": update_families()["permutation_mirror"], "translation_2^20": build(24, shift=2.0 ** 20)}


def world_soup(inst, blasses):
    """every instance's triangles moved to world space in fp64 -> (tri (m, 3, 3), offset of each instance, each triangle's instance
    translation length)"""
    out, offs, shift, o = [], [], [], 0
    for x in inst:
        v = blasses[int(x["blasIdx"])][2].reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
        M = x["transform"].astype(np.float64).reshape(4, 4)
        out.append(v @ M[:3, :3].T + M[:3, 3])
        shift.append(np.full(v.shape[0], np.linalg.norm(M[:3, 3])))
        offs.append(o)
        o += v.shape[0]
    return np.concatenate(out), np.array(offs, np.int64), np.concatenate(shift)


def world_rays(tri, n, seed):
    """n rays from uniform points of the world box in random directions, tmax inf"""
    rng = np.random.default_rng(seed)
    lo, hi = tri.reshape(-1, 3).min(0), tri.reshape(-1, 3).max(0)
    O = (lo + rng.uniform(0, 1, (n, 3)) * (hi - lo)).astype(np.float32)
    return R.gpu_records(R.make_rays(O, rng.normal(size=(n, 3)).astype(np.float32), np.float32(np.inf)))


def tlas_scene(name):
    from oracle import refpy
    from tests.test_intersect_all_tlas import host_tlas, port_blasses
    T = affine_families()[name]
    v = [scenes.procedural_scene(400, 3), scenes.procedural_scene(300, 4)]
    inst = refpy.make_instances(T, np.arange(T.shape[0]) % 2)
    blasses = port_blasses(v)
    tn, ti = host_tlas(inst, blasses)
    tri, offs, shift = world_soup(inst, blasses)
    return tn, ti, inst, blasses, tri, offs, shift


def tlas_rules(tri, offs, shift, rays, h, ii, c, k=K):
    """the rules on a two-level result: a record is the world triangle of its (instance, prim); the ray is moved to BLAS space in fp32
    through the instance's inverse, so t is held to 1e-6 of the larger of |O - v0| and max( |O|, the instance's translation ) over the
    cosine of the ray's angle to the normal, over |D|, and the edge margin is the coordinate ulps over that cosine"""
    p = ao.prims(h).astype(np.int64)
    flat = np.where(ii == ao.NO_PRIM, 0, offs[np.minimum(ii, offs.shape[0] - 1)] + np.where(p == ao.NO_PRIM, 0, p))
    mag = np.maximum(np.linalg.norm(rays["O"].astype(np.float64), axis=1)[:, None], shift[None])
    return check_rules(rays, tri, h, c, k, p=flat, mag=mag)


@pytest.mark.parametrize("name", ["rigid", "nonuniform_scale", "permutation_mirror", "translation_2^20"])
def test_tlas_affine_instances(name):
    """the world ray against every instance's triangles moved to world space in fp64: t is shared between world and BLAS space"""
    from tests import allhits_tlas_oracle as tao
    tn, ti, inst, blasses, tri, offs, shift = tlas_scene(name)
    rays = world_rays(tri, 200, 5)
    h, ii, c, _ = tao.brute(tn, ti, inst, blasses, rays, K)
    res = tlas_rules(tri, offs, shift, rays, h, ii, c)
    print(name, res)
    assert_rules(res, name)
