"""The host restatement of the multi-hit ray query (tests/allhits_oracle.c, DESIGN.md §4.14), without a GPU: the definition over every
reached reference against the pruned walk (and the walk in reverse child order) on trees of every builder, the uploaded-tree families,
a DAG, a failed-split SBVH and golden, flat, signed-zero and scaled scenes; k = 1 against BVH::Intersect's t, count > 0 against
BVH::IsOccluded, SBVH split triangles once, saturation at k + 1, the NaN-t and tmax rules, and ray parity against an fp64 winding number
on closed icospheres."""
import os

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import rays as R, scenes
from tests import allhits_oracle as ao, util
from tests.test_closest_point import builder_trees, family

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_PRIM = ao.NO_PRIM
KS = (1, 2, 4, 5, 16, 17, 63, 64)


def rays_for(v, rng, n=600):
    """camera rays, rays from inside and around the box in random directions, rays started on triangles, axis and octant rays, the same
    with a user rD of +-inf, and a mix of tmax: BVH_FAR, inf, finite, 0, negative and NaN"""
    tri = v.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    lo, hi = scenes.scene_bounds(v)
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    ext = float((hi - lo).max()) or 1.0
    eye, view = R.bounds_camera(lo, hi, "outside")
    parts = [R.primary_rays(eye, view, 16, 16, 1)]
    mid = (lo + hi) / 2
    O = mid + rng.uniform(-1, 1, (n, 3)) * (hi - lo + ext * 0.1)
    parts.append(R.make_rays(O.astype(np.float32), rng.normal(size=(n, 3)).astype(np.float32)))
    k = rng.integers(0, tri.shape[0], n // 2)
    w = rng.dirichlet((1, 1, 1), n // 2)
    on = (w[:, :, None] * tri[k]).sum(1)
    parts.append(R.make_rays(on.astype(np.float32), rng.normal(size=(n // 2, 3)).astype(np.float32)))
    ax = util.axis_rays(lo, hi, 4, seed=int(rng.integers(1 << 30)))
    oc = util.octant_rays(lo, hi, 16, seed=int(rng.integers(1 << 30)))
    parts += [ax, oc, util.with_inf_rd(ax), util.with_inf_rd(oc)]
    r = np.concatenate(parts)
    sel = rng.integers(0, 8, r.shape[0])
    t = np.choose(sel, [np.full(r.shape[0], R.BVH_FAR), np.full(r.shape[0], np.inf), rng.uniform(0, 2 * ext, r.shape[0]),
                        rng.uniform(0, 0.3 * ext, r.shape[0]), np.zeros(r.shape[0]), np.full(r.shape[0], R.BVH_FAR),
                        np.full(r.shape[0], -1.0), np.full(r.shape[0], np.nan)]).astype(np.float32)
    r["t"] = t
    return R.gpu_records(r)


def same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def check_same(nodes, idx, v, rays, label, ks=(1, 4, 17, 64)):
    """brute == walk == reverse walk, byte for byte, for every k; returns the brute results of the largest k"""
    out = None
    for k in ks:
        h, c, keys = ao.brute(nodes, idx, v, rays, k)
        wh, wc = ao.walk(nodes, idx, v, rays, k)
        assert same(h, wh) and np.array_equal(c, wc), f"{label} k={k}: pruned walk differs from the definition"
        rh, rc = ao.walk(nodes, idx, v, rays, k, reverse=True)
        assert same(h, rh) and np.array_equal(c, rc), f"{label} k={k}: the walk depends on its child order"
        assert (c <= k + 1).all()
        p = ao.prims(h)
        filled = np.arange(k)[None, :] < np.minimum(c, k)[:, None]
        assert np.array_equal(p != NO_PRIM, filled), f"{label} k={k}: records past the count"
        out = (h, c, keys)
    return out


@pytest.mark.parametrize("ntris", [1, 7, 2000])
def test_brute_force_equals_pruned_walk(ntris):
    v = scenes.procedural_scene(ntris, 11 + ntris)
    rays = rays_for(v, np.random.default_rng(ntris))
    for label, nodes, idx in builder_trees(v):
        check_same(nodes, idx, v, rays, f"{label}-{ntris}")


def test_failed_split_sbvh_brute_force_equals_pruned_walk():
    """an SBVH whose spatial splits fail: leaves built from stale idxTmp words need not hold their triangles"""
    from tests.test_build_hq_shapes import fail_scene, fail_scene_hq
    v = fail_scene("snapped3k_q4")
    nodes, idx = fail_scene_hq("snapped3k_q4")[:2]
    check_same(nodes, idx, v, rays_for(v, np.random.default_rng(6)), "snapped3k_q4")


@pytest.mark.parametrize("fam", util.FAMILIES + ["shrunk", "dag"])
def test_families_brute_force_equals_pruned_walk(fam):
    v = scenes.procedural_scene(3000, 71)
    src = util.source_tree(v, "BuildHQ" if fam in ("A1", "DB") else "Build")
    nodes, idx = family(src, fam)
    check_same(nodes, idx, v, rays_for(v, np.random.default_rng(9), n=400), fam)


@pytest.mark.parametrize("name", ["flat_500", "coincident_610", "single_tri", "atrium_3k"])
def test_golden_scenes(name):
    g = np.load(os.path.join(REPO, "tests", "golden", f"{name}.npz"))
    v = g["verts"].astype(np.float32)
    nodes = np.ascontiguousarray(g["nodes"]).view(portpy.NODE32).reshape(-1)
    check_same(nodes, g["prim_idx"], v, rays_for(v, np.random.default_rng(10), n=400), name)


@pytest.mark.parametrize("variant", ["zero-random", "zero-order", "scale2^-20", "scale2^20"])
def test_signed_zero_and_scaled_scenes(variant):
    v = scenes.procedural_scene(2000, 33)
    if variant.startswith("zero"):
        v = util.signed_zero(v, variant[5:])
    else:
        v = util.scaled(v, int(variant.split("^")[1]))
    for label, nodes, idx in builder_trees(v)[:3]:
        check_same(nodes, idx, v, rays_for(v, np.random.default_rng(11), n=400), f"{variant}/{label}", ks=(1, 5, 64))


def test_k1_and_count_match_intersect_and_occluded():
    """k = 1: record 0's t is BVH::Intersect's bit for bit wherever its key is its t, and its prim differs only on an exact-t tie;
    count > 0 is BVH::IsOccluded's bit"""
    v = scenes.procedural_scene(3000, 5)
    rays = rays_for(v, np.random.default_rng(3), n=1500)
    # a user rD of +-inf makes NaN slab terms, which the reference's min / max keep and the engine's drop (DESIGN.md 4.1)
    rays = rays[np.isfinite(rays["rD"]).all(1)]
    for label, nodes, idx in builder_trees(v):
        h, c, keys = ao.brute(nodes, idx, v, rays, 1)
        host = np.zeros(rays.shape[0], R.RAY_DTYPE)
        host.view(np.uint8).reshape(-1, 128)[:, :64] = rays.view(np.uint8).reshape(-1, 64)
        o = portpy.PortBVH(v, nodes=nodes, prim_idx=idx)
        ref = o.intersect(host.copy())
        occ = o.occluded(host)
        bit = np.unpackbits(occ.view(np.uint8), bitorder="little")[: rays.shape[0]].astype(bool)
        assert np.array_equal(c > 0, bit), f"{label}: count > 0 differs from IsOccluded"
        hit = c > 0
        exact = hit & (keys[:, 0].view(np.uint32) == h[:, 0, 0].view(np.uint32))
        assert exact.sum() > 0.9 * hit.sum()
        assert same(h[exact, 0, 0], ref["t"][exact]), f"{label}: t differs from Intersect where key == t"
        diff = exact & (ao.prims(h)[:, 0] != ref["prim"])
        for i in np.nonzero(diff)[0]:
            # a tie: Intersect's own triangle is accepted at the same t
            hh, cc, _ = ao.brute(nodes, idx, v, rays[i:i + 1], 64)
            ts = hh[0, : min(int(cc[0]), 64), 0]
            ps = ao.prims(hh)[0, : min(int(cc[0]), 64)]
            assert ref["prim"][i] in ps[ts == h[i, 0, 0]], f"{label}: ray {i} differs from Intersect without a tie"


def test_sbvh_split_triangles_once():
    """BuildHQ references a split triangle from several leaves: it appears in a ray's records once, and the count counts it once"""
    v = scenes.procedural_scene(3000, 71)
    nodes, idx, _ = portpy.build_hq(v)
    assert idx.shape[0] > v.shape[0] // 3, "the scene has no split triangles"
    rays = rays_for(v, np.random.default_rng(2), n=1500)
    h, c, _ = ao.brute(nodes, idx, v, rays, 64)
    p = ao.prims(h)
    for i in range(rays.shape[0]):
        got = p[i, : min(int(c[i]), 64)]
        assert np.unique(got).shape[0] == got.shape[0], f"ray {i}: a prim twice"
    # against one leaf holding every triangle once: never more (a split triangle counted twice would be), and the same count on nearly
    # every ray (the SBVH's clipped boxes may miss a crossing on their boundary planes in fp32, such as a ray started on a triangle)
    lone = np.zeros(2, portpy.NODE32)
    lone[0] = (v.reshape(-1, 4)[:, :3].min(0), 0, v.reshape(-1, 4)[:, :3].max(0), v.shape[0] // 3)
    one = ao.brute(lone, np.arange(v.shape[0] // 3, dtype=np.uint32), v, rays, 64)[1]
    assert (c <= one).all(), "a split triangle counted more than once"
    assert (c == one).mean() > 0.97


def test_saturation_and_order():
    """a ray through m parallel layers: count = min( m, k + 1 ), records nearest first, the rest empty"""
    m = 12
    z = np.arange(m, dtype=np.float32) + 1
    tri = np.zeros((m, 3, 4), np.float32)
    tri[:, 0, :3] = np.stack([np.full(m, -1), np.full(m, -1), z], 1)
    tri[:, 1, :3] = np.stack([np.full(m, 3), np.full(m, -1), z], 1)
    tri[:, 2, :3] = np.stack([np.full(m, -1), np.full(m, 3), z], 1)
    v = tri[::-1].reshape(-1, 4).copy()   # prim 0 is the farthest layer
    o = portpy.PortBVH(v)
    rays = R.gpu_records(R.make_rays(np.array([[0, 0, 0]], np.float32), np.array([[0, 0, 1]], np.float32)))
    for k in (1, 4, 11, 12, 13, 64):
        h, c, _ = ao.brute(o.nodes, o.prim_idx, v, rays, k)
        assert int(c[0]) == min(m, k + 1)
        n = min(m, k)
        assert np.array_equal(h[0, :n, 0], z[:n]) and np.array_equal(ao.prims(h)[0, :n], m - 1 - np.arange(n))
        assert (ao.prims(h)[0, n:] == NO_PRIM).all() and (h[0, n:, 0] == R.BVH_FAR).all() and (h[0, n:, 1:3] == 0).all()
    # tmax between layers 5 and 6 keeps five; tmax exactly on a layer keeps it
    for t, want in ((5.5, 5), (6.0, 6), (0.5, 0)):
        r = rays.copy()
        r["t"] = t
        h, c, _ = ao.brute(o.nodes, o.prim_idx, v, r, 64)
        assert int(c[0]) == want and (h[0, want:, 0] == np.float32(t)).all()


def test_tmax_and_nan_rules():
    """tmax NaN or negative: count 0 and records { tmax, 0, 0, NO_PRIM }; tmax 0 keeps only hits at t == 0; a hit whose t is NaN (huge
    coordinates overflowing the triangle test) is not accepted, where BVH::Intersect's own test would take it"""
    v = scenes.procedural_scene(500, 3)
    o = portpy.PortBVH(v)
    rays = rays_for(v, np.random.default_rng(4), n=200)
    h, c, _ = ao.brute(o.nodes, o.prim_idx, v, rays, 4)
    bad = np.isnan(rays["t"]) | (rays["t"] < 0)
    assert bad.any() and (c[bad] == 0).all()
    assert same(h[bad, :, 0], np.repeat(rays["t"][bad, None], 4, 1)) and (ao.prims(h)[bad] == NO_PRIM).all()
    zero = rays["t"] == 0
    assert (h[zero & (c > 0), 0, 0] == 0).all()
    # NaN t: a triangle at 1e30 scale crossed by a ray whose direction makes f * dot overflow to inf - inf
    big = np.float32(3e38)
    tri = np.array([[-big, -big, big, 0], [big, -big, big, 0], [0, big, big, 0]], np.float32)
    tri2 = np.array([[-1, -1, 1, 0], [1, -1, 1, 0], [0, 1, 1, 0]], np.float32)
    v2 = np.concatenate([tri, tri2])
    one = np.zeros(2, portpy.NODE32)
    one[0] = ((-big, -big, 1), 0, (big, big, big), 2)
    ray = R.gpu_records(R.make_rays(np.array([[0, 0, 0]], np.float32), np.array([[0, 0, 1]], np.float32), np.float32(np.inf)))
    h, c, _ = ao.brute(one, np.arange(2, dtype=np.uint32), v2, ray, 4)
    assert not np.isnan(h[0, :, 0]).any(), "a NaN t was accepted"


def fp64_winding(V, F, p):
    """the fp64 winding number of the closed mesh (V, F) at points p (van Oosterom & Strackee's solid angle)"""
    a, b, c = (V[F[:, j]][None, :, :] - p[:, None, :] for j in range(3))
    la, lb, lc = (np.linalg.norm(x, axis=2) for x in (a, b, c))
    det = np.einsum("ijk,ijk->ij", a, np.cross(b, c))
    den = la * lb * lc + np.einsum("ijk,ijk->ij", a, b) * lc + np.einsum("ijk,ijk->ij", b, c) * la + np.einsum("ijk,ijk->ij", c, a) * lb
    return (2 * np.arctan2(det, den)).sum(1) / (4 * np.pi)


def test_ray_parity_on_closed_icospheres():
    """k = 64 on closed icospheres: wherever count <= 64, count parity says inside exactly when the fp64 winding number does, except rays
    that cross within rounding of an edge (min( u, v, 1 - u - v ) < 1e-5 on some record: two neighbours both or neither accepted)"""
    from tests.test_signed_distance import icosphere
    parts = []
    for sub, r, c in ((2, 1.0, (0, 0, 0)), (3, 0.6, (2.5, 0.3, -0.2)), (1, 0.3, (-1.7, 1.1, 0.9))):
        V, F = icosphere(sub, r, c)
        parts.append((V, F))
    Vs = np.concatenate([p[0] for p in parts])
    offs = np.cumsum([0] + [p[0].shape[0] for p in parts])[:-1]
    Fs = np.concatenate([p[1] + o for p, o in zip(parts, offs)])
    v = np.zeros((Fs.shape[0] * 3, 4), np.float32)
    v[:, :3] = Vs[Fs].reshape(-1, 3)
    rng = np.random.default_rng(12)
    n = 3000
    O = rng.uniform(-2.5, 3.5, (n, 3)).astype(np.float32)
    rays = R.gpu_records(R.make_rays(O, rng.normal(size=(n, 3)).astype(np.float32), np.float32(np.inf)))
    Vf = v.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    Vw, Fw = Vf.reshape(-1, 3), np.arange(Vf.shape[0] * 3).reshape(-1, 3)
    wn = fp64_winding(Vw, Fw, O.astype(np.float64))
    inside = wn > 0.5
    for label, nodes, idx in builder_trees(v):
        h, c, _ = ao.brute(nodes, idx, v, rays, 64)
        ok = c <= 64
        odd = (c % 2) == 1
        wrong = np.nonzero(ok & (odd != inside))[0]
        for i in wrong:
            m = int(c[i])
            u, vv = h[i, :m, 1].astype(np.float64), h[i, :m, 2].astype(np.float64)
            edge = np.minimum(np.minimum(u, vv), 1 - u - vv).min() if m else np.inf
            print(f"{label}: ray {i} count {m} winding {wn[i]:.6f} nearest edge {edge:.3g}")
            assert edge < 1e-5, f"{label}: ray {i} parity disagrees with the winding number away from an edge"
        assert len(wrong) <= n // 100, f"{label}: {len(wrong)} parity exceptions"
