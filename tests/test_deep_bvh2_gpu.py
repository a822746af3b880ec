"""BVH2 trees 64 to 256 levels deep, and the depth every producer reports.

The BVH2 walk picks its stack from `info.max_depth`: the 64-entry kernels below depth 64, the same kernels with the reference's
256-entry stack (tiny_bvh.h:3249) from 64 to 255, TBVH_E_LIMIT above.  A BLAS under a TLAS is walked with a 64-entry stack, so a
BVH-layout BLAS of depth 64 or more is refused.  No builder makes trees that deep from the seeded scenes, so the deep walks run on
hand-encoded spines: every inner node holds one inner child and one one-triangle leaf, and a ray down the spine axis pushes one
leaf per level, `depth` stack entries at the bottom.

Any-hit: the reference's IsOccluded stack holds 64 entries (tiny_bvh.h:3409); the plain-C restatement's holds 256.  Beyond depth
64 the engine's any-hit walk is held to the restatement, not to the reference.

`info.max_depth` is what keeps a per-ray stack from overflowing, so it is held equal to the depth of the downloaded tree for
every producer: the builders and their settings, uploads, refits, the TLAS build and a group replica."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from tinybvh_b200 import _lib, api, rays as R, scenes
from oracle import portpy
from tests import util

F = np.float32
YZ_LO, YZ_HI = F(-1), F(3)          # every leaf triangle spans y, z in [-1, 3]; spine rays run near y = z = 0
DEPTHS = [1, 62, 63, 64, 65, 128, 255]


# ---- the spine -------------------------------------------------------------------------------------------------------------

def is_tie_level(k, depth):
    """Levels whose leaf has exactly the inner sibling's box (equal entry distance for every ray): the left-on-ties rule decides."""
    return k % 5 == 3 and k < depth - 1


def spine(depth, seed=0):
    """-> (nodes NODE32[2 + 2 * depth], primIdx, verts): a BVH2 of exactly `depth` in the reference's layout (node 1 unused, sibling
    pairs).  Inner node I_k (k = 0 .. depth-1, I_0 the root) has the children I_(k+1) and leaf L_k; I_(depth-1) has the leaves
    L_(depth-1) and L_depth.  Leaf L_k holds one real triangle in the plane x = X_k, with X_depth = 0 and X increasing towards the
    root by seeded steps, so the leaf lies beyond its inner sibling along +x.  On tie levels (is_tie_level) L_k holds a slanted
    triangle whose box is exactly the box of I_(k+1), and I_(k+1) is the left child.  Elsewhere the leaf takes the left slot on odd
    levels and the right slot on even ones.  Every box is the union of its children's.  Prim numbers are a seeded permutation."""
    assert depth >= 1
    rng = np.random.default_rng(seed)
    perm = rng.permutation(depth + 1).astype(np.uint32)
    steps = (8 + rng.integers(0, 17, depth + 1)).astype(np.float32) / F(16)   # 0.5 .. 1.5 in 1/16: sums stay exact
    tri = np.zeros((depth + 1, 3, 3), np.float32)

    def plane(x):
        return np.array([[x, YZ_LO, YZ_LO], [x, YZ_HI, YZ_LO], [x, YZ_LO, YZ_HI]], np.float32)

    tri[depth] = plane(F(0))
    tri[depth - 1] = plane(steps[depth - 1])
    lo = tri[depth - 1:].reshape(-1, 3).min(0)
    hi = tri[depth - 1:].reshape(-1, 3).max(0)
    box = [None] * depth            # box of I_k
    box[depth - 1] = (lo, hi)
    for k in range(depth - 2, -1, -1):
        blo, bhi = box[k + 1]
        if is_tie_level(k, depth):
            tri[k] = [[blo[0], blo[1], blo[2]], [bhi[0], bhi[1], blo[2]], [blo[0], blo[1], bhi[2]]]
        else:
            tri[k] = plane(F(bhi[0] + steps[k]))
        box[k] = (np.minimum(blo, tri[k].min(0)), np.maximum(bhi, tri[k].max(0)))
    nodes = np.zeros(2 + 2 * depth, portpy.NODE32)
    verts = np.zeros((3 * (depth + 1), 4), np.float32)
    verts.reshape(-1, 3, 4)[perm, :, :3] = tri

    def put(i, b, left_first, count):
        nodes[i]["aabbMin"], nodes[i]["aabbMax"], nodes[i]["leftFirst"], nodes[i]["triCount"] = b[0], b[1], left_first, count

    def leaf_box(k):
        return tri[k].min(0), tri[k].max(0)

    put(0, box[0], 2, 0)
    for k in range(depth):
        pair = 2 + 2 * k
        leaf_slot = 1 if is_tie_level(k, depth) else k % 2 ^ 1
        if k + 1 < depth:
            put(pair + (leaf_slot ^ 1), box[k + 1], pair + 2, 0)
        else:
            put(pair + (leaf_slot ^ 1), leaf_box(depth), depth, 1)
        put(pair + leaf_slot, leaf_box(k), k, 1)
    return nodes, perm.copy(), verts


def bvh2_depth(nodes):
    """Depth of the deepest node (root = 0) of a NODE32 tree: leaves are the nodes with triCount > 0."""
    frontier, depth = np.zeros(1, np.int64), 0
    while True:
        inner = frontier[nodes["triCount"][frontier] == 0]
        if inner.size == 0:
            return depth
        first = nodes["leftFirst"][inner].astype(np.int64)
        frontier, depth = np.concatenate([first, first + 1]), depth + 1


def bvh_gpu_depth(nodes):
    """Depth of a NODE64 (BVH_GPU) tree: inner nodes have triCount 0 and name both children."""
    frontier, depth = np.zeros(1, np.int64), 0
    while True:
        inner = frontier[nodes["triCount"][frontier] == 0]
        if inner.size == 0:
            return depth
        frontier, depth = np.concatenate([nodes["left"][inner], nodes["right"][inner]]).astype(np.int64), depth + 1


def walk(nodes, prim_idx, verts, ray, anyhit=False):
    """The kernel's walk of one ray in float64 (enough for the spine's well-separated planes; equal boxes still tie exactly):
    -> (hit prim or None, deepest stack, node visits, triangle tests)."""
    O, D, rD = (ray[f].astype(np.float64) for f in ("O", "D", "rD"))
    tmax, prim = float(ray["t"]), None
    v = verts.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    stack, deepest, steps, tris = [], 0, 0, 0
    node = nodes[0]
    ref, cnt = int(node["leftFirst"]), int(node["triCount"])
    while True:
        steps += 1
        if cnt == 0:
            ab = []
            for c in (nodes[ref], nodes[ref + 1]):
                t1, t2 = (c["aabbMin"] - O) * rD, (c["aabbMax"] - O) * rD
                tn, tf = max(np.minimum(t1, t2).max(), 0.0), min(np.maximum(t1, t2).min(), tmax)
                ab.append((tf >= tn, tn, int(c["leftFirst"]), int(c["triCount"])))
            (ha, ta, ra, ca), (hb, tb, rb, cb) = ab
            if ha and hb:
                if ta > tb:
                    (ref, cnt), push = (rb, cb), (ra, ca)
                else:
                    (ref, cnt), push = (ra, ca), (rb, cb)
                stack.append(push)
                deepest = max(deepest, len(stack))
                continue
            if ha or hb:
                ref, cnt = (ra, ca) if ha else (rb, cb)
                continue
        else:
            for j in range(ref, ref + cnt):
                p = int(prim_idx[j])
                tris += 1
                v0, e1, e2 = v[p, 0], v[p, 1] - v[p, 0], v[p, 2] - v[p, 0]
                h = np.cross(D, e2)
                a = e1 @ h
                if abs(a) < 1e-7:
                    continue
                s = O - v0
                u = (s @ h) / a
                q = np.cross(s, e1)
                w = (D @ q) / a
                t = (e2 @ q) / a
                if u >= 0 and w >= 0 and u + w <= 1 and 0 <= t <= tmax:
                    tmax, prim = t, p
                    if anyhit:
                        return prim, deepest, steps, tris
        if not stack:
            return prim, deepest, steps, tris
        ref, cnt = stack.pop()


def spine_rays(nodes, count, seed):
    """Rays down the spine, `count` per direction octant: +x octants start at x = -1 and walk the whole chain, -x octants start
    past the root box and meet the top leaf first.  Small y / z direction components carry the octant's signs."""
    rng = np.random.default_rng(seed)
    x_hi = F(nodes[0]["aabbMax"][0])
    O, D = [], []
    for s in util.octant_dirs():
        o = np.zeros((count, 3), np.float32)
        o[:, 0] = F(-1) if s[0] > 0 else x_hi + F(1)
        o[:, 1:] = (rng.random((count, 2)) - 0.5).astype(np.float32)
        d = np.ones((count, 3), np.float32) * s
        d[:, 1:] *= (F(1e-4) + rng.random((count, 2)).astype(np.float32) * F(4e-4))
        O.append(o), D.append(d)
    return R.make_rays(np.concatenate(O), np.concatenate(D))


def forward_spine_rays(rays):
    return rays[rays["D"][:, 0] > 0]


def spine_ray_set(nodes, seed):
    """Spine rays of every octant, rays from inside the chain's box in random directions, and misses (above the box, and pointing
    away from it), in uniform-octant and mixed warps."""
    lo, hi = nodes[0]["aabbMin"], nodes[0]["aabbMax"]
    sp = spine_rays(nodes, 36, seed)
    rnd = util.octant_rays(lo, hi, 24, seed)
    rng = np.random.default_rng(seed + 1)
    o = np.zeros((48, 3), np.float32)
    o[:, 0] = -1
    o[:24, 1] = 10 + rng.random(24).astype(np.float32)
    d = np.zeros((48, 3), np.float32)
    d[:24, 0], d[24:, 0] = 1, -1
    d[:, 1:] = (rng.random((48, 2)) - 0.5).astype(np.float32) * F(1e-3)
    return util.octant_blocks(np.concatenate([sp, rnd, R.make_rays(o, d)]), seed)


# ---- CPU checks of the spine ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("depth", [1, 2, 5, 62, 63, 64, 65, 128, 255, 256])
def test_spine_is_what_it_claims(depth):
    nodes, idx, verts = spine(depth, seed=depth)
    assert bvh2_depth(nodes) == depth
    assert nodes.shape[0] == 2 + 2 * depth and (nodes[1].tobytes() == bytes(32))
    v = verts.reshape(-1, 3, 4)[:, :, :3]
    ties = 0
    for k in range(depth):
        a, b = nodes[2 + 2 * k], nodes[3 + 2 * k]
        parent = nodes[0] if k == 0 else [n for n in nodes[2 * k:2 * k + 2] if n["triCount"] == 0][0]
        assert np.array_equal(parent["aabbMin"], np.minimum(a["aabbMin"], b["aabbMin"])), f"level {k}: box is not the union"
        assert np.array_equal(parent["aabbMax"], np.maximum(a["aabbMax"], b["aabbMax"])), f"level {k}: box is not the union"
        inner = int(a["triCount"] == 0) + int(b["triCount"] == 0)
        assert inner == (1 if k + 1 < depth else 0), f"level {k}: {inner} inner children"
        for c in (a, b):
            if c["triCount"]:
                p = idx[c["leftFirst"]]
                assert c["triCount"] == 1
                assert np.array_equal(c["aabbMin"], v[p].min(0)) and np.array_equal(c["aabbMax"], v[p].max(0)), f"level {k}: leaf box"
        if k + 1 < depth:
            ties += a.tobytes()[:12] == b.tobytes()[:12] and a.tobytes()[16:28] == b.tobytes()[16:28]
    assert ties == sum(is_tie_level(k, depth) for k in range(depth))
    if depth > 2:
        assert {int(nodes[2 + 2 * k]["triCount"] > 0) for k in range(depth - 1)} == {0, 1}, "leaves sit in both slots"
    assert sorted(idx.tolist()) == list(range(depth + 1))
    # the walk down the spine: depth stack entries, every node visited, the deepest leaf's triangle (the nearest) closest
    last = int(idx[[n["leftFirst"] for n in nodes[2 * depth:] if n["aabbMax"][0] == 0][0]])
    for ray in forward_spine_rays(spine_rays(nodes, 2, depth))[::2]:
        prim, deepest, steps, tris = walk(nodes, idx, verts, ray)
        assert (prim, deepest, steps, tris) == (last, depth, 2 * depth + 1, depth + 1)
        prim, deepest, steps, tris = walk(nodes, idx, verts, ray, anyhit=True)
        assert (prim, deepest, steps, tris) == (last, depth, depth + 1, 1)
    if depth <= 255:   # the restatement's stack holds 256 entries: never walk a deeper tree with it
        r = forward_spine_rays(spine_rays(nodes, 8, depth))
        want = r.copy()
        portpy.PortBVH(verts, nodes=nodes, prim_idx=idx).intersect(want)
        assert (want["prim"] == last).all()


def test_python_walk_notices_the_tie_rule():
    """On a tie level the left (inner) child is entered first; entering the leaf first would let its hit cull the next plane leaf."""
    nodes, idx, verts = spine(10, 3)
    ray = forward_spine_rays(spine_rays(nodes, 1, 3))[0]
    swapped = nodes.copy()
    for k in range(10):
        if is_tie_level(k, 10):
            swapped[[2 + 2 * k, 3 + 2 * k]] = swapped[[3 + 2 * k, 2 + 2 * k]]
    assert bvh2_depth(swapped) == 10
    assert walk(swapped, idx, verts, ray)[2] < walk(nodes, idx, verts, ray)[2] == 21


# ---- GPU: walks at depths 1 .. 255 -------------------------------------------------------------------------------------------

def engine(layout, nodes, idx, verts):
    if layout == "BVH":
        return api.BVH().upload(nodes, idx, verts)
    return api.BVH_GPU().upload(portpy.PortBVH(verts, nodes=nodes, prim_idx=idx).to_bvh_gpu(), idx, verts)


@pytest.fixture(scope="module", params=DEPTHS)
def deep_case(request):
    depth = request.param
    nodes, idx, verts = spine(depth, seed=depth)
    r = spine_ray_set(nodes, depth)
    o = portpy.PortBVH(verts, nodes=nodes, prim_idx=idx)
    want = r.copy()
    o.intersect(want)
    s = r.copy()
    k = np.arange(r.shape[0]) % 3
    s["t"] = np.where(k == 0, R.BVH_FAR, np.where(k == 1, want["t"], want["t"] * F(0.5))).astype(np.float32)
    occ = np.unpackbits(o.occluded(s).view(np.uint8), bitorder="little")[: r.shape[0]].astype(bool)
    return depth, nodes, idx, verts, r, want, s, occ


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["BVH", "BVH_GPU"])
def test_deep_walk_matches_oracle(gpu, deep_case, layout):
    """Closest and any-hit walks at depths 1 .. 255 under trace_variant 0, 3 and 4, statistics on and off, from host records,
    128-byte device records in place and 64-byte records with a 16-byte hit array, for 1, 31, 33, all-but-37 and all rays: bit for
    bit the restatement's walk; occlusion bits past n zero, the word after (n+31)/32 untouched; statistics the same for every
    shape and variant."""
    from tests.test_hot_path_gpu import assert_hits, pack, run_anyhit, run_closest, unpack, SENTINEL
    depth, nodes, idx, verts, r, want, s, occ = deep_case
    e = engine(layout, nodes, idx, verts)
    assert e.info().max_depth == depth
    hit = want["t"] < R.BVH_FAR
    assert hit.sum() > r.shape[0] // 3 and (~hit).sum() >= 48 and occ.any() and not occ.all()
    full = r.shape[0]
    try:
        for n in (1, 31, 33, full - 37, full):
            stats = {"closest": set(), "any": set()}
            for variant in (0, 3, 4):
                api.set_option("trace_variant", variant)
                for st in (False, True):
                    e.set_stats(st)
                    label = f"depth {depth} {layout} n={n} trace_variant {variant} stats {st}"
                    h = r[:n].copy()
                    e.Intersect(h)
                    assert util.compare_hits(h, want[:n]) == {"prim": 0, "t": 0, "u": 0, "v": 0}, f"{label} host"
                    if st:
                        stats["closest"].add(e.get_stats())
                    for shape in ("64+hits", "128"):
                        assert_hits(run_closest(e, r, n, shape), want[:n], f"{label} {shape}", need_hit=False)
                        if st:
                            stats["closest"].add(e.get_stats())
                    bits = np.full((n + 31) // 32 + 1, SENTINEL, np.uint32)
                    e.IsOccluded(s[:n].copy(), bits=bits)
                    assert bits[-1] == SENTINEL, f"{label} host: the word after (n+31)/32 was written"
                    assert np.array_equal(bits[:-1], pack(occ[:n])), f"{label} host any-hit: {(unpack(bits[:-1], n) != occ[:n]).sum()} bits differ"
                    if st:
                        stats["any"].add(e.get_stats())
                    for stride in (64, 128):
                        got = run_anyhit(e, s, n, stride)
                        assert np.array_equal(got, pack(occ[:n])), f"{label} {stride}-byte any-hit: {(unpack(got, n) != occ[:n]).sum()} bits differ"
                        if st:
                            stats["any"].add(e.get_stats())
            assert len(stats["closest"]) == 1 and len(stats["any"]) == 1, f"depth {depth} n={n}: statistics differ: {stats}"
    finally:
        e.set_stats(False)
        api.set_option("trace_variant", 3)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["BVH", "BVH_GPU"])
def test_deep_walk_statistics_are_the_closed_form(gpu, deep_case, layout):
    """Rays down the spine visit every node (2 * depth + 1) and test every leaf's triangle (depth + 1) for the closest hit, and stop
    at the deepest leaf (depth + 1 visits, one test) for the any-hit query: the order of the walk, ties included, is the
    reference's.  The hits are the deepest leaf's triangle."""
    depth, nodes, idx, verts = deep_case[:4]
    e = engine(layout, nodes, idx, verts)
    r = forward_spine_rays(spine_rays(nodes, 64, depth + 1))
    n = r.shape[0]
    last = walk(nodes, idx, verts, r[0])[0]
    e.set_stats(True)
    try:
        got = r.copy()
        e.Intersect(got)
        assert e.get_stats()[:2] == (n * (2 * depth + 1), n * (depth + 1))
        assert (got["prim"] == last).all()
        assert e.IsOccluded(r.copy()).tolist() == [0xFFFFFFFF] * (n // 32)
        assert e.get_stats()[:2] == (n * (depth + 1), n)
    finally:
        e.set_stats(False)


# ---- limits -----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["BVH", "BVH_GPU"])
def test_depth_256_is_refused(gpu, layout):
    """One level past the 256-entry stack: every walk is refused with TBVH_E_LIMIT before a launch, and no ray record or bit word
    changes.  (The restatement is never run on this tree: its own 256-entry stack would overflow.)"""
    import torch
    nodes, idx, verts = spine(256, 256)
    e = engine(layout, nodes, idx, verts)
    assert e.info().max_depth == 256
    r = spine_ray_set(nodes, 256)
    h = r.copy()
    with pytest.raises(api.TbvhError, match="depth 256 exceeds"):
        e.Intersect(h)
    assert h.tobytes() == r.tobytes()
    bits = np.full((r.shape[0] + 31) // 32, 0x5A5A5A5A, np.uint32)
    with pytest.raises(api.TbvhError, match="depth 256 exceeds"):
        e.IsOccluded(r.copy(), bits=bits)
    assert (bits == 0x5A5A5A5A).all()
    for stride in (64, 128):
        d = torch.from_numpy(np.ascontiguousarray(r.view(np.uint8).reshape(-1, 128)[:, :stride])).cuda()
        before = d.cpu().numpy()
        hits = torch.full((r.shape[0], 4), float("nan"), dtype=torch.float32, device="cuda") if stride == 64 else None
        with pytest.raises(api.TbvhError, match="depth 256 exceeds"):
            e.Intersect(d, hits=hits)
        db = torch.full((bits.shape[0],), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        with pytest.raises(api.TbvhError, match="depth 256 exceeds"):
            e.IsOccluded(d, bits=db)
        torch.cuda.synchronize()
        assert np.array_equal(d.cpu().numpy(), before)
        assert (db.cpu().numpy() == 0x5A5A5A5A).all()
        if hits is not None:
            assert torch.isnan(hits).all()


def instances():
    """Identity, mirror (x -> -x) and rotation-and-scale instances of one BLAS, 40 units apart in z."""
    inst = np.zeros(3, api.BLAS_INSTANCE)
    m = [np.eye(4, dtype=np.float32), np.diag([-1, 1, 1, 1]).astype(np.float32), util.random_transforms(1, 17, spread=0)[0].reshape(4, 4)]
    for i in range(3):
        m[i][2, 3] += F(40 * i)
        inst[i]["transform"] = m[i].reshape(-1)
        inst[i]["mask"] = 0xFFFF
    return inst


def world_rays(inst, nodes, seed):
    """Spine rays of every octant carried into world space by each instance's transform, and random rays through the world boxes."""
    out = []
    for i in range(inst.shape[0]):
        m = inst[i]["transform"].reshape(4, 4).astype(np.float64)
        r = spine_rays(nodes, 16, seed + i)
        out.append(R.make_rays((r["O"] @ m[:3, :3].T + m[:3, 3]).astype(np.float32), (r["D"] @ m[:3, :3].T).astype(np.float32)))
        out.append(util.octant_rays(inst[i]["aabbMin"], inst[i]["aabbMax"], 8, seed + i))
    return util.octant_blocks(np.concatenate(out), seed)


@pytest.mark.gpu
def test_tlas_over_blas_of_depth_63(gpu):
    """The deepest BVH-layout BLAS the two-level walk takes: 63 pushes into its 64-entry stack.  TLAS tree, hits and occlusion bits
    are the restatement's (BVH::Build over the instance boxes, IntersectTLAS / IsOccludedTLAS) bit for bit."""
    from tests.test_tlas_gpu import words
    nodes, idx, verts = spine(63, 63)
    blas = api.BVH().upload(nodes, idx, verts)
    assert blas.info().max_depth == 63
    inst = instances()
    inst_ref = inst.copy()
    ref = util._PortTLAS(inst_ref, [portpy.PortBVH(verts, nodes=nodes, prim_idx=idx)])
    t = api.TLAS().Build(inst, [blas])
    assert inst.tobytes() == inst_ref.tobytes()
    tn, ti = t.download()
    assert np.array_equal(tn.view(np.uint32), ref.tree.nodes.view(np.uint32)) and np.array_equal(ti, ref.tree.prim_idx)
    rays = world_rays(inst, nodes, 5)
    want, got = rays.copy(), rays.copy()
    ref.intersect(want), t.Intersect(got)
    assert np.array_equal(words(got), words(want))
    assert (want["t"] < R.BVH_FAR).sum() > rays.shape[0] // 2 and set(want["pad"][want["t"] < R.BVH_FAR]) == {0, 1, 2}
    s = rays.copy()
    s["t"] = np.where(np.arange(s.shape[0]) % 2 == 0, want["t"], want["t"] * F(0.5))
    assert np.array_equal(t.IsOccluded(s), ref.occluded(s))


@pytest.mark.gpu
def test_tlas_refuses_bvh_blas_of_depth_64(gpu):
    nodes, idx, verts = spine(64, 64)
    blas = api.BVH().upload(nodes, idx, verts)
    with pytest.raises(api.TbvhError, match="BLAS 0 has depth 64"):
        api.TLAS().Build(instances(), [blas])


@pytest.mark.gpu
def test_tlas_over_deep_blas_holding_its_cwbvh(gpu):
    """A BLAS of depth 64 that also holds its CWBVH: the TLAS is built, its CWBVH walk matches the restatement's composition
    (IntersectTLAS with BVH8_CWBVH::Intersect per instance), and a walk through the BVH layout is refused with the depth."""
    from tests.test_tlas_gpu import words
    nodes, idx, verts = spine(64, 64)
    blas = api.BVH().upload(nodes, idx, verts)
    api.check(_lib.lib().tbvh_convert(blas.h, api.LAYOUT_CWBVH))
    inst = instances()
    t = api.TLAS().Build(inst, [blas], blas_layout=api.LAYOUT_CWBVH)
    tn, ti = t.download()
    port = portpy.PortTLASCW(tn, ti, inst, [cw_bytes(blas)])
    rays = world_rays(inst, nodes, 7)
    want, got = rays.copy(), rays.copy()
    port.intersect(want), t.Intersect(got)
    assert np.array_equal(words(got), words(want)) and (want["t"] < R.BVH_FAR).sum() > rays.shape[0] // 2
    s = rays.copy()
    s["t"] = np.where(np.arange(s.shape[0]) % 2 == 0, R.BVH_FAR, want["t"] * F(0.5))
    assert np.array_equal(t.IsOccluded(s), port.occluded(s))
    t.layout = api.LAYOUT_BVH
    with pytest.raises(api.TbvhError, match="BLAS 0 has depth 64"):
        t.Intersect(rays.copy())
    with pytest.raises(api.TbvhError, match="BLAS 0 has depth 64"):
        t.IsOccluded(rays.copy())


# ---- a CWBVH from a deep BVH2 ----------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("depth", [63, 64, 200])
def test_cwbvh_of_a_deep_spine(gpu, depth):
    """tbvh_convert of the uploaded spine on the device: the walk is bit for bit the restatement's BVH8_CWBVH::Intersect over the
    downloaded bytes, and the wide tree needs at most 128 pending node groups.  (The reference's SplitLeafs stack holds 64 entries,
    so there is no byte oracle for the conversion of these trees, and the restatement's converter is never run on them.)"""
    from tests.test_hot_path_gpu import assert_hits, to_device
    import torch
    nodes, idx, verts = spine(depth, depth)
    e = api.BVH().upload(nodes, idx, verts)
    api.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_CWBVH))
    e.layout = api.LAYOUT_CWBVH
    cw = cw_bytes(e)
    assert util.cw_depth_and_pending(cw.nodes)[1] <= 128
    r = spine_ray_set(nodes, depth)
    want = r.copy()
    portpy.PortCWBVH.intersect(cw, want)
    assert (want["t"] < R.BVH_FAR).sum() > r.shape[0] // 3
    got = r.copy()
    e.Intersect(got)
    assert util.compare_hits(got, want) == {"prim": 0, "t": 0, "u": 0, "v": 0}
    hits = torch.empty((r.shape[0], 4), dtype=torch.float32, device="cuda")
    e.Intersect(to_device(r), hits=hits)
    assert_hits(hits.cpu().numpy(), want, f"CWBVH depth {depth} 64+hits", need_hit=False)
    s = r.copy()
    s["t"] = np.where(np.arange(s.shape[0]) % 2 == 0, R.BVH_FAR, want["t"] * F(0.5))
    occ = s["t"] > portpy.PortCWBVH.intersect(cw, s.copy())["t"]
    from tests.test_hot_path_gpu import pack
    assert np.array_equal(e.IsOccluded(s), pack(occ))


# ---- info.max_depth of every producer ---------------------------------------------------------------------------------------

def cw_bytes(e):
    """bvh8Data / bvh8Tris of a handle, for the restatement's BVH8_CWBVH::Intersect (portpy.PortCWBVH.intersect, PortTLASCW)."""
    d8, t8 = api.BVH8_CWBVH.download(e)
    return SimpleNamespace(nodes=d8, tris=t8)


def downloaded_depth(e):
    return bvh2_depth(api.BVH.download(e)[0])


def assert_depth(e, label):
    """info.max_depth is exactly the depth of the tree the handle holds, and of its BVH_GPU form when it has one."""
    i = e.info()
    got = downloaded_depth(e)
    assert i.max_depth == got, f"{label}: info.max_depth {i.max_depth}, downloaded tree depth {got}"
    if i.layouts & (1 << api.LAYOUT_BVH_GPU):
        assert bvh_gpu_depth(api.BVH_GPU.download(e)) == got, f"{label}: BVH_GPU depth"
    return got


BUILDERS = ["Build", "BuildAVX", "BuildHQ"]


@pytest.mark.gpu
@pytest.mark.parametrize("ntris", [1, 2, 3, 31, 257, 5000, 70000, 400000])
@pytest.mark.parametrize("builder", BUILDERS)
def test_builders_report_their_depth(gpu, builder, ntris):
    v = scenes.procedural_scene(ntris, 11)
    e = getattr(api.BVH(), builder)(v)
    d = assert_depth(e, f"{builder} {ntris}")
    assert d > 0 or ntris < 3
    # the same triangles through the indexed overload
    if ntris in (31, 5000, 70000):
        verts, ind = np.unique(v.reshape(-1, 4), axis=0, return_inverse=True)
        x = getattr(api.BVH(), builder)(verts, indices=ind.astype(np.uint32).reshape(-1))
        assert x.info().max_depth == d == downloaded_depth(x), f"{builder} {ntris} indexed"


@pytest.mark.gpu
@pytest.mark.parametrize("build_mode", [0, 1])
@pytest.mark.parametrize("small_t", [8, 64, 256])
@pytest.mark.parametrize("builder", ["Build", "BuildAVX"])
def test_build_settings_report_their_depth(gpu, builder, small_t, build_mode):
    """The switch point to the per-warp small-subtree kernel and both drivers of the large phase."""
    try:
        api.set_option("small_t", small_t)
        api.set_option("build_mode", build_mode)
        for ntris in (300, 70000):
            e = getattr(api.BVH(), builder)(scenes.procedural_scene(ntris, 13))
            assert_depth(e, f"{builder} small_t {small_t} build_mode {build_mode} {ntris}")
    finally:
        api.set_option("small_t", 128)
        api.set_option("build_mode", 0)


@pytest.mark.gpu
@pytest.mark.parametrize("costs", [(1.0, 1.0), (0.25, 4.0), (8.0, 0.5)])
@pytest.mark.parametrize("builder", BUILDERS)
def test_sah_constants_report_their_depth(gpu, builder, costs):
    e = api.BVH()
    e.c_trav, e.c_int = costs
    getattr(e, builder)(scenes.procedural_scene(20000, 17))
    assert_depth(e, f"{builder} c_trav/c_int {costs}")


FAMILIES = ["scale:90", "scale:60", "scale:-126", "scale:40", "shift:-12582912", "zero:order", "leaf:identical", "leaf:clusters", "leaf:collapsed"]


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("builder", BUILDERS)
def test_offatrium_families_report_their_depth(gpu, builder, fam):
    """Scales where every SAH cost overflows (the root split into two leaves, or kept as a leaf with its range rotated: depth 1 or
    0), tiny and translated scenes, signed zeros, and the long-leaf families."""
    from tests.test_offatrium_gpu import family
    kind, arg = fam.split(":")
    for ntris in (3, 2000):
        v = util.long_leaf_scene(arg) if kind == "leaf" else family(fam, ntris)
        assert_depth(getattr(api.BVH(), builder)(v), f"{builder} {fam} {ntris}")
        if kind == "leaf":
            break


def derived(cls, builder, v):
    """A BVH_GPU / BVH8_CWBVH handle over the tree BVH.<builder> makes (their Build is BuildAVX's flavour unless told otherwise)."""
    h = cls()
    if builder == "BuildHQ":
        return h.BuildHQ(v)
    h.build_flavour = _lib.BUILD_REFERENCE if builder == "Build" else _lib.BUILD_AVX
    return h.Build(v)


@pytest.mark.gpu
@pytest.mark.parametrize("builder", BUILDERS)
def test_derived_handles_report_their_depth(gpu, builder):
    """The BVH2 a BVH8_CWBVH / BVH_GPU handle keeps, the BVH and BVH_GPU uploads of a built tree, refits, a TLAS and a group
    replica: each reports the depth of the tree it holds."""
    from tests.test_oracle_pin import moved
    v = scenes.procedural_scene(30000, 19)
    e = getattr(api.BVH(), builder)(v)
    d = assert_depth(e, f"BVH.{builder}")
    cw, g = derived(api.BVH8_CWBVH, builder, v), derived(api.BVH_GPU, builder, v)
    assert assert_depth(cw, f"BVH8_CWBVH {builder}") == d and assert_depth(g, f"BVH_GPU {builder}") == d
    nodes, idx = e.download()
    gn = api.BVH_GPU.download(g)
    up = api.BVH_GPU().upload(gn, idx, v)
    assert up.info().max_depth == bvh_gpu_depth(gn) == d
    assert assert_depth(api.BVH().upload(nodes, idx, v), "BVH upload") == d
    if builder != "BuildHQ":   # BVH::Refit refuses an SBVH
        w = moved(v, 3, amp=0.05)
        e.Refit(w)
        assert assert_depth(e, "Refit") == d
        cw.Refit(w)
        assert assert_depth(cw, "BVH8_CWBVH refit_layouts") == d
        g.Refit(w)
        assert assert_depth(g, "BVH_GPU refit_layouts") == d
    from tests.test_oracle_pin import tlas_case
    tv, inst, _, _ = tlas_case(91, 300)
    t = api.TLAS().Build(inst, [getattr(api.BVH(), builder)(x) for x in tv])
    assert_depth(t, "TLAS")
    grp = api.Group([0, 0])
    try:
        grp.replicate(e)
        for k in range(len(grp)):
            rep = _lib.lib().tbvh_group_replica(grp.h, k)
            i = _lib.Info()
            api.check(_lib.lib().tbvh_bvh_info(C.c_void_p(rep), C.byref(i)))
            rn = np.zeros(i.used_nodes, api.NODE32)
            api.check(_lib.lib().tbvh_download_bvh(C.c_void_p(rep), rn.ctypes.data, None, api.HOST))
            assert i.max_depth == bvh2_depth(rn) == d, f"group replica {k}"
    finally:
        grp.close()
