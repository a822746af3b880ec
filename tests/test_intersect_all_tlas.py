"""The host restatement of multi-hit rays through a TLAS (tests/allhits_tlas_oracle.c, DESIGN.md §4.14 two levels), without a GPU: the definition
over every reached reference against the pruned walk, in both child and instance orders, on TLAS scenes of 1, 40 and 300 instances under
two ray masks, BLASses of every builder (BuildHQ's split triangles included), the uploaded-tree families and a DAG, the instance-update
transform families and one BLAS instanced many times; the anchors: a one-instance identity TLAS is the single-level query with instance 0,
two instances under one transform give every hit twice, k = 1 against IntersectTLAS / IsOccludedTLAS, and ray parity over rigid instances
of a closed icosphere."""
import numpy as np
import pytest

from oracle import portpy, refpy
from tinybvh_b200 import rays as R, scenes
from tests import allhits_oracle as ao, allhits_tlas_oracle as tao, util
from tests.test_closest_point import builder_trees, family
from tests.test_intersect_all import fp64_winding, rays_for, same
from tests.test_oracle_pin import tlas_case
from tests.test_tlas_update import update_families

NO_PRIM = ao.NO_PRIM


def host_tlas(inst, blasses):
    """BLASInstance::Update of every record (in place) and the TLAS over the instance boxes, as util's port TLAS builds it -> (nodes,
    prim_idx).  blasses: (nodes, prim_idx, verts) per BLAS."""
    lo = np.stack([b[0][0]["aabbMin"] for b in blasses])[inst["blasIdx"]]
    hi = np.stack([b[0][0]["aabbMax"] for b in blasses])[inst["blasIdx"]]
    with np.errstate(all="ignore"):
        portpy.instance_update(inst, lo, hi)
    fake = np.zeros((inst.shape[0] * 3, 4), np.float32)
    fake[0::3, :3], fake[1::3, :3], fake[2::3, :3] = inst["aabbMin"], inst["aabbMax"], inst["aabbMin"]
    t = portpy.PortBVH(fake)
    return t.nodes, t.prim_idx


def tlas_rays(inst, rng, n=400, mask=0xFFFF):
    """camera rays onto the instances' world box, rays from inside and around it in random directions, axis and octant rays, the same
    with a user rD of +-inf, and a mix of tmax: BVH_FAR, inf, finite, 0, negative and NaN"""
    lo, hi = inst["aabbMin"].astype(np.float64), inst["aabbMax"].astype(np.float64)
    ok = np.isfinite(lo).all(1) & np.isfinite(hi).all(1) & (lo <= hi).all(1)
    lo, hi = (lo[ok].min(0), hi[ok].max(0)) if ok.any() else (np.full(3, -1.0), np.full(3, 1.0))
    lo, hi = np.maximum(lo, -1e30).astype(np.float32), np.minimum(hi, 1e30).astype(np.float32)
    ext = float((hi.astype(np.float64) - lo).max()) or 1.0
    eye, view = R.bounds_camera(lo, hi, "outside")
    parts = [R.primary_rays(eye, view, 12, 12, 1)]
    mid = (lo.astype(np.float64) + hi) / 2
    O = mid + rng.uniform(-0.6, 0.6, (n, 3)) * (hi.astype(np.float64) - lo)
    parts.append(R.make_rays(O.astype(np.float32), rng.normal(size=(n, 3)).astype(np.float32)))
    ax = util.axis_rays(lo, hi, 3, seed=int(rng.integers(1 << 30)))
    oc = util.octant_rays(lo, hi, 8, seed=int(rng.integers(1 << 30)))
    parts += [ax, oc, util.with_inf_rd(ax), util.with_inf_rd(oc)]
    r = np.concatenate(parts)
    m = r.shape[0]
    sel = rng.integers(0, 8, m)
    t = np.choose(sel, [np.full(m, R.BVH_FAR), np.full(m, np.inf), rng.uniform(0, 2 * ext, m), rng.uniform(0, 0.3 * ext, m), np.zeros(m),
                        np.full(m, R.BVH_FAR), np.full(m, -1.0), np.full(m, np.nan)]).astype(np.float32)
    r["t"] = t
    r["mask"] = mask
    return R.gpu_records(r)


def check_same(tn, ti, inst, blasses, rays, label, ks=(1, 4, 17, 64)):
    """brute == walk == reverse walk, byte for byte, for every k; returns the brute results of the largest k"""
    out = None
    for k in ks:
        h, ii, c, keys = tao.brute(tn, ti, inst, blasses, rays, k)
        for rev in (False, True):
            wh, wi, wc = tao.walk(tn, ti, inst, blasses, rays, k, reverse=rev)
            assert same(h, wh) and np.array_equal(ii, wi) and np.array_equal(c, wc), \
                f"{label} k={k}: the {'reverse ' if rev else ''}pruned walk differs from the definition"
        assert (c <= k + 1).all()
        filled = np.arange(k)[None, :] < np.minimum(c, k)[:, None]
        assert np.array_equal(ao.prims(h) != NO_PRIM, filled) and np.array_equal(ii != NO_PRIM, filled), f"{label} k={k}: records past the count"
        out = (h, ii, c, keys)
    return out


def port_blasses(vs, builder=0):
    return [(t[1], t[2], v) for v, t in ((v, builder_trees(v)[builder]) for v in vs)]


@pytest.mark.parametrize("n_inst", [1, 40, 300])
@pytest.mark.parametrize("mask", [0x1, 0x2])
def test_tlas_cases(n_inst, mask):
    v, inst, O, D = tlas_case(91, n_inst)
    blasses = port_blasses(v)
    tn, ti = host_tlas(inst, blasses)
    rays = tlas_rays(inst, np.random.default_rng(n_inst), n=300, mask=mask)
    h, ii, c, _ = check_same(tn, ti, inst, blasses, rays, f"{n_inst}/{mask:#x}")
    seen = np.unique(ii[ii != NO_PRIM])
    if n_inst > 1:
        assert seen.shape[0] > 1
    # a mask-0x1 ray never sees an instance that carries 0x2 only (every fifth)
    assert mask == 0x2 or not np.isin(seen, np.arange(0, n_inst, 5)).any()


@pytest.mark.parametrize("builder", [0, 1, 2, 3])
def test_builders(builder):
    """BLASses from Build, BuildAVX, BuildHQ (split triangles: one prim from several leaves) and BuildPLOC"""
    v, inst, O, D = tlas_case(92, 40)
    blasses = port_blasses(v, builder)
    tn, ti = host_tlas(inst, blasses)
    check_same(tn, ti, inst, blasses, tlas_rays(inst, np.random.default_rng(7), n=300, mask=0x2), f"builder {builder}")


@pytest.mark.parametrize("fam", util.FAMILIES + ["shrunk", "dag"])
def test_uploaded_families(fam):
    v = scenes.procedural_scene(3000, 71)
    src = util.source_tree(v, "BuildHQ" if fam in ("A1", "DB") else "Build")
    nodes, idx = family(src, fam)
    inst = refpy.make_instances(util.random_transforms(20, 5), [0] * 20)
    blasses = [(nodes, idx, v)]
    tn, ti = host_tlas(inst, blasses)
    check_same(tn, ti, inst, blasses, tlas_rays(inst, np.random.default_rng(9), n=250), fam, ks=(1, 5, 64))


@pytest.mark.parametrize("name", list(update_families().keys()))
def test_update_families(name):
    """permutation and mirror, singular, projective, 2^+-60 scales and a 2^20 translation: the transforms the instance update and the ray
    transform are sensitive to"""
    T = update_families()[name]
    v = [scenes.procedural_scene(500, 3), scenes.procedural_scene(300, 4)]
    inst = refpy.make_instances(T, np.arange(T.shape[0]) % 2)
    blasses = port_blasses(v)
    tn, ti = host_tlas(inst, blasses)
    check_same(tn, ti, inst, blasses, tlas_rays(inst, np.random.default_rng(3), n=250), name, ks=(1, 4, 17, 64))


def test_one_blas_instanced_many_times():
    v = scenes.procedural_scene(800, 12)
    inst = refpy.make_instances(util.random_transforms(500, 6, spread=30.0), [0] * 500)
    blasses = port_blasses([v])
    tn, ti = host_tlas(inst, blasses)
    h, ii, c, _ = check_same(tn, ti, inst, blasses, tlas_rays(inst, np.random.default_rng(4), n=300), "500 instances", ks=(2, 16, 63))
    assert np.unique(ii[ii != NO_PRIM]).shape[0] > 50


def identity_tlas(v, copies=1):
    inst = refpy.make_instances(np.tile(np.eye(4, dtype=np.float32).reshape(1, 16), (copies, 1)), [0] * copies)
    blasses = port_blasses([v])
    return (*host_tlas(inst, blasses), inst, blasses)


def test_identity_instance_is_the_single_level_query():
    """a one-instance identity TLAS gives orc_ah_brute's records with instance 0, on rays whose rD is safercp( D ) and whose O and D hold no
    -0 (the transform's sums turn a -0 into +0, which may flip the sign of a zero u or v)"""
    v = scenes.procedural_scene(3000, 5)
    tn, ti, inst, blasses = identity_tlas(v)
    rays = rays_for(v, np.random.default_rng(8), n=800)
    negzero = lambda a: (a.view(np.uint32) == 0x80000000).any(1)
    rays = rays[(rays["rD"].view(np.uint32) == R.safercp(rays["D"]).view(np.uint32)).all(1) & ~negzero(rays["O"]) & ~negzero(rays["D"])]
    assert rays.shape[0] > 1500
    for k in (1, 4, 17, 64):
        h, ii, c, keys = tao.brute(tn, ti, inst, blasses, rays, k)
        want = ao.brute(blasses[0][0], blasses[0][1], v, rays, k)
        assert same(h, want[0]) and np.array_equal(c, want[1]) and same(keys, want[2]), f"k={k}"
        filled = np.arange(k)[None, :] < np.minimum(c, k)[:, None]
        assert (ii[filled] == 0).all() and (ii[~filled] == NO_PRIM).all()


def test_two_instances_under_one_transform_give_every_hit_twice():
    v = scenes.procedural_scene(2000, 6)
    T = util.random_transforms(1, 3, spread=2.0)
    one = refpy.make_instances(T, [0])
    two = refpy.make_instances(np.concatenate([T, T]), [0, 0])
    blasses = port_blasses([v])
    t1, i1 = host_tlas(one, blasses)
    t2, i2 = host_tlas(two, blasses)
    rays = tlas_rays(one, np.random.default_rng(5), n=600)
    h1, ii1, c1, _ = tao.brute(t1, i1, one, blasses, rays, 32)
    h2, ii2, c2, _ = check_same(t2, i2, two, blasses, rays, "two copies", ks=(64,))
    assert np.array_equal(c2, np.minimum(2 * c1, 65))
    m = np.minimum(c1, 32)
    for j in range(32):
        rows = m > j
        for s, want_inst in ((2 * j, 0), (2 * j + 1, 1)):
            assert same(h2[rows, s], h1[rows, j]) and (ii2[rows, s] == want_inst).all(), f"slot {s}"
    assert (c1 > 0).sum() > 100


def test_k1_and_count_match_intersect_tlas_and_occluded_tlas():
    """k = 1: record 0's t is IntersectTLAS's bit for bit wherever key == t, its instance and prim differ only on exact-t ties; count > 0
    is IsOccludedTLAS's bit (rays with a NaN tmax or a NaN t aside)"""
    v, inst, O, D = tlas_case(94, 60)
    blasses = port_blasses(v)
    tn, ti = host_tlas(inst, blasses)
    port = portpy.PortTLAS(tn, ti, inst, [portpy.PortBVH(b[2], nodes=b[0], prim_idx=b[1]) for b in blasses])
    for mask in (0x1, 0x2):
        rays = tlas_rays(inst, np.random.default_rng(mask), n=1500, mask=mask)
        rays = rays[np.isfinite(rays["rD"]).all(1) & ~np.isnan(rays["t"])]
        h, ii, c, keys = tao.brute(tn, ti, inst, blasses, rays, 1)
        host = np.zeros(rays.shape[0], R.RAY_DTYPE)
        host.view(np.uint8).reshape(-1, 128)[:, :64] = rays.view(np.uint8).reshape(-1, 64)
        ref = port.intersect(host.copy())
        occ = np.unpackbits(port.occluded(host).view(np.uint8), bitorder="little")[: rays.shape[0]].astype(bool)
        nan_t = np.isnan(ref["t"])
        assert np.array_equal((c > 0)[~nan_t], occ[~nan_t]), f"mask {mask:#x}: count > 0 differs from IsOccludedTLAS"
        # key > t where a leaf box's entry distance rounds above the triangle's t: more often in BLAS space, where tight leaf boxes meet
        # transformed rays (about a quarter of the hits here)
        exact = (c > 0) & (keys[:, 0].view(np.uint32) == h[:, 0, 0].view(np.uint32))
        assert exact.sum() > 0.6 * (c > 0).sum() and exact.sum() > 200
        assert same(h[exact, 0, 0], ref["t"][exact]), f"mask {mask:#x}: t differs from IntersectTLAS where key == t"
        diff = exact & ((ao.prims(h)[:, 0] != ref["prim"]) | (ii[:, 0] != ref["pad"]))
        for i in np.nonzero(diff)[0]:
            hh, hi, cc, _ = tao.brute(tn, ti, inst, blasses, rays[i:i + 1], 64)
            m = min(int(cc[0]), 64)
            at = hh[0, :m, 0] == h[i, 0, 0]
            pairs = set(zip(hi[0, :m][at].tolist(), ao.prims(hh)[0, :m][at].tolist()))
            assert (int(ref["pad"][i]), int(ref["prim"][i])) in pairs, f"ray {i} differs from IntersectTLAS without a tie"


def rigid_transforms(n, seed, spread):
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 16), np.float32)
    for i in range(n):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        a, b, c, d = q
        m = np.eye(4)
        m[:3, :3] = [[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]]
        m[:3, 3] = rng.uniform(-spread, spread, 3)
        out[i] = m.astype(np.float32).reshape(-1)
    return out


def test_ray_parity_over_rigid_icosphere_instances():
    """k = 64, infinite tmax, rigid instances of one closed icosphere: wherever count <= 64 its parity is the parity of the number of
    instances whose fp64 winding number at the ray origin says inside, except rays that cross within 1e-5 of an edge"""
    from tests.test_signed_distance import icosphere
    V, F = icosphere(2, 1.0, (0, 0, 0))
    v = np.zeros((F.shape[0] * 3, 4), np.float32)
    v[:, :3] = V[F].reshape(-1, 3)
    T = rigid_transforms(24, 9, 1.5)
    inst = refpy.make_instances(T, [0] * 24)
    blasses = port_blasses([v])
    tn, ti = host_tlas(inst, blasses)
    rng = np.random.default_rng(13)
    n = 2000
    O = rng.uniform(-2.5, 2.5, (n, 3)).astype(np.float32)
    rays = R.gpu_records(R.make_rays(O, rng.normal(size=(n, 3)).astype(np.float32), np.float32(np.inf)))
    Vf = v.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    Vw, Fw = Vf.reshape(-1, 3), np.arange(Vf.shape[0] * 3).reshape(-1, 3)
    inside = np.zeros(n, np.int64)
    for t in T.astype(np.float64).reshape(-1, 4, 4):
        p = (np.linalg.inv(t) @ np.concatenate([O.astype(np.float64), np.ones((n, 1))], 1).T).T[:, :3]
        inside += fp64_winding(Vw, Fw, p) > 0.5
    h, ii, c, _ = tao.brute(tn, ti, inst, blasses, rays, 64)
    ok = c <= 64
    wrong = np.nonzero(ok & ((c % 2) != (inside % 2)))[0]
    for i in wrong:
        m = int(c[i])
        u, vv = h[i, :m, 1].astype(np.float64), h[i, :m, 2].astype(np.float64)
        edge = np.minimum(np.minimum(u, vv), 1 - u - vv).min() if m else np.inf
        assert edge < 1e-5, f"ray {i}: parity disagrees with the instances containing its origin away from an edge"
    assert len(wrong) <= n // 100 and (inside > 0).sum() > 100 and (c > 0).mean() > 0.3
