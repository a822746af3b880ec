"""Shared helpers for the parity tests: oracle selection, ray sets, comparators."""
import numpy as np

from tinybvh_b200 import rays as R, scenes
from oracle import portpy, refpy


def oracle_bvh(verts):
    """The parity oracle for a triangle soup: the compiled reference (BVH::Build + Intersect/IsOccluded) when
    oracle/_ref exists, else the pinned plain-C restatement.  Both expose .nodes/.prim_idx/.intersect/.occluded."""
    if refpy.available():
        return refpy.RefBVH(verts, mode=0, threaded=False)
    return portpy.PortBVH(verts)


def oracle_tree(verts, mode=0):
    """The reference's BVH::Build (mode 0), BuildAVX (1) or BuildHQ (2) tree, single-threaded numbering: the compiled reference when
    oracle/_ref exists, else the pinned restatements (tests/test_oracle_pin.py).  -> .nodes/.prim_idx/.idx_count/.intersect/.occluded."""
    if refpy.available():
        return refpy.RefBVH(verts, mode=mode, threaded=False)
    if mode == 2:
        nodes, idx, ic = portpy.build_hq(verts)
        o = portpy.PortBVH(verts, nodes=nodes, prim_idx=idx)
    else:
        o = portpy.PortBVH(verts, avx=mode == 1)
        ic = o.prim_idx.shape[0]
    o.idx_count = ic
    return o


def oracle_bvh_gpu_nodes(tree):
    """BVH_GPU::ConvertFrom of an oracle_tree()."""
    return refpy.RefBVHGPU(tree).nodes if refpy.available() else tree.to_bvh_gpu()


def oracle_cwbvh(verts, mode=2):
    """BVH8_CWBVH data + the reference's CPU walk of it.  mode as refpy.RefCWBVH: 0 Build (over BuildAVX), 1 BuildHQ, 2 the Build chain
    over the scalar BVH::Build tree.  Without oracle/_ref: the pinned conversion chain over the pinned tree (test_port_cwbvh_matches_*).
    -> (cwbvh with .nodes/.tris/.intersect, number of referenced bvh8Tris records)"""
    if refpy.available():
        cw = refpy.RefCWBVH(verts, mode=mode)
        return cw, int(cw.source_bvh().nodes["triCount"].sum()) * 3
    b = oracle_tree(verts, {0: 1, 1: 2, 2: 0}[mode])
    used = int(b.nodes["triCount"].sum())
    return portpy.PortCWBVH(b.nodes, b.prim_idx[:used], verts, idx_count=b.idx_count), used * 3


class _PortTLAS:
    """BVH::Build( BLASInstance*, .. ) + IntersectTLAS / IsOccludedTLAS from the pinned restatements (test_port_tlas_matches_golden_vectors):
    Update()s the instances in place, builds the TLAS over their boxes, walks it with the BLASses."""

    def __init__(self, inst, blasses):
        lo = np.stack([b.nodes[0]["aabbMin"] for b in blasses])[inst["blasIdx"]]
        hi = np.stack([b.nodes[0]["aabbMax"] for b in blasses])[inst["blasIdx"]]
        portpy.instance_update(inst, lo, hi)
        # a "triangle" (min, max, min) has exactly the instance's box
        fake = np.zeros((inst.shape[0] * 3, 4), np.float32)
        fake[0::3, :3], fake[1::3, :3], fake[2::3, :3] = inst["aabbMin"], inst["aabbMax"], inst["aabbMin"]
        self.tree = portpy.PortBVH(fake)
        self.port = portpy.PortTLAS(self.tree.nodes, self.tree.prim_idx, inst, blasses)

    def intersect(self, rays, threads=0):
        return self.port.intersect(rays)

    def occluded(self, rays, threads=0):
        return self.port.occluded(rays)

    def bvh(self):
        return self.tree


def oracle_tlas(inst, verts_list, mode=0):
    """The reference's TLAS over BLASses built with oracle_tree(mode); Update()s `inst` in place.  -> .intersect/.occluded/.bvh()"""
    blasses = [oracle_tree(v, mode) for v in verts_list]
    if refpy.available():
        return refpy.RefTLAS(inst, blasses)
    return _PortTLAS(inst, blasses)


def renumber_bfs(nodes):
    """The same BVH2 with its sibling pairs numbered breadth-first (root 0, unused node 1 kept): a tree whose node order is not the
    builder's, as a multi-threaded build leaves it."""
    nodes = np.ascontiguousarray(nodes)
    order, k = [0, 1], 0
    while k < len(order):
        i = order[k]
        k += 1
        if i != 1 and nodes[i]["triCount"] == 0:
            order += [int(nodes[i]["leftFirst"]), int(nodes[i]["leftFirst"]) + 1]
    pos = np.zeros(nodes.shape[0], np.int64)
    pos[order] = np.arange(len(order))
    out = nodes[order].copy()
    inner = out["triCount"] == 0
    inner[1] = False
    out["leftFirst"][inner] = pos[out["leftFirst"][inner]]
    return out


# ---- trees no builder makes: the same triangles under other valid BVH2s, for the consumers of an uploaded tree
# Every family keeps node 1 unused, children behind their parent (BVH::Refit walks the nodes backwards) and every primIdx entry a
# valid triangle number.  A tree is (nodes NODE32, primIdx[idx_count], idx_count).

def source_tree(verts, builder):
    """BVH::Build / BuildAVX / BuildHQ of a scene as an uploadable tree: primIdx padded with zeros to idxCount (the SBVH's tail)."""
    o = oracle_tree(verts, {"Build": 0, "BuildAVX": 1, "BuildHQ": 2}[builder])
    ic = int(getattr(o, "idx_count", o.prim_idx.shape[0]))
    idx = np.zeros(ic, np.uint32)
    idx[: o.prim_idx.shape[0]] = o.prim_idx
    return np.ascontiguousarray(o.nodes).view(portpy.NODE32).reshape(-1).copy(), idx, ic


def optimized_tree(verts, iterations=25):
    """BVH::Build followed by the reference's own BVH::Optimize (needs oracle/_ref): the tree the shim's BVH::Optimize uploads."""
    o = refpy.RefBVH.optimized(verts, iterations)
    return np.ascontiguousarray(o.nodes).view(portpy.NODE32).reshape(-1).copy(), o.prim_idx.copy(), int(o.idx_count)


def tree_levels(nodes):
    """-> list of node-index arrays per depth (root = level 0), over the nodes reachable from the root."""
    frontier, out = np.zeros(1, np.int64), []
    while frontier.size:
        out.append(frontier)
        inner = frontier[nodes["triCount"][frontier] == 0]
        first = nodes["leftFirst"][inner].astype(np.int64)
        frontier = np.stack([first, first + 1], 1).reshape(-1)
    return out


def tree_depth(nodes):
    return len(tree_levels(nodes)) - 1


def dfs_leaves(nodes):
    """-> leaf node indices in DFS order (left child first)."""
    out, stack = [], [0]
    lf, tc = nodes["leftFirst"], nodes["triCount"]
    while stack:
        x = stack.pop()
        if tc[x]:
            out.append(x)
        else:
            stack += [int(lf[x]) + 1, int(lf[x])]
    return np.array(out, np.int64)


def leaf_order_is_dfs(nodes):
    """True when firstTri grows along the DFS leaf order: the order every builder leaves and BVH_GPU::ConvertFrom's old closed form
    assumed."""
    f = nodes["leftFirst"][dfs_leaves(nodes)].astype(np.int64)
    return bool((np.diff(f) > 0).all())


def refold_boxes(nodes):
    """Interior boxes recomputed bottom-up from the leaf boxes with the reference's tinybvh_min / tinybvh_max (a < b ? a : b,
    a > b ? a : b; left child first), in place."""
    for lvl in reversed(tree_levels(nodes)):
        inner = lvl[nodes["triCount"][lvl] == 0]
        if inner.size == 0:
            continue
        c = nodes["leftFirst"][inner].astype(np.int64)
        lmin, rmin = nodes["aabbMin"][c], nodes["aabbMin"][c + 1]
        lmax, rmax = nodes["aabbMax"][c], nodes["aabbMax"][c + 1]
        nodes["aabbMin"][inner] = np.where(lmin < rmin, lmin, rmin)
        nodes["aabbMax"][inner] = np.where(lmax > rmax, lmax, rmax)
    return nodes


def swapped(tree, seed, frac):
    """Family A: the two child records of a seeded share `frac` of the interior nodes exchanged (at least one; frac = 1 mirrors the
    tree).  Numbering, boxes and primIdx stay; the DFS leaf order changes."""
    nodes, idx, ic = tree
    nodes = nodes.copy()
    inner = np.concatenate(tree_levels(nodes))
    inner = inner[nodes["triCount"][inner] == 0]
    if inner.size:
        rng = np.random.default_rng(seed)
        pick = rng.permutation(inner)[: max(1, int(round(frac * inner.size)))]
        c = nodes["leftFirst"][pick].astype(np.int64)
        nodes[c], nodes[c + 1] = nodes[c + 1].copy(), nodes[c].copy()
    return nodes, idx.copy(), ic


def write_dfs(nodes, left, right, root):
    """A tree given as child lists written back as BVH::ConvertFrom( BVH_Verbose ) writes it: DFS preorder, the k-th interior node's
    children at 2 + 2k and 3 + 2k, leaves keep firstTri / triCount / box; interior boxes refolded."""
    out = np.zeros(nodes.shape[0], portpy.NODE32)
    nxt, stack = 2, [(root, 0)]
    while stack:
        s, d = stack.pop()
        if left[s] < 0:
            out[d] = nodes[s]
            continue
        out[d]["leftFirst"], out[d]["triCount"] = nxt, 0
        stack += [(right[s], nxt + 1), (left[s], nxt)]
        nxt += 2
    assert nxt == nodes.shape[0], "the tree has holes"
    return refold_boxes(out)


def reinserted(tree, seed, k, max_depth=63, grow_to=None):
    """Family B, the shape BVH::Optimize leaves: k seeded subtree reinsertions.  Subtree X leaves its parent P, X's sibling takes
    P's place, and P becomes the parent of X and a node Y outside X's subtree (in either slot order).  A reinsertion that would
    make the tree deeper than max_depth is not made.  grow_to: Y is the deepest leaf and X a leaf off its path, until the tree is
    that deep (the 64..255 range of the 256-entry walk).  Written back in ConvertFrom( BVH_Verbose )'s numbering; leaves keep
    firstTri, so the DFS leaf order no longer follows primIdx (more reinsertions are made until it does not)."""
    nodes, idx, ic = tree
    rng = np.random.default_rng(seed)
    n = nodes.shape[0]
    left, right, parent, height = [-1] * n, [-1] * n, [-1] * n, [0] * n
    levels = tree_levels(nodes)
    for lvl in reversed(levels):
        for x in lvl.tolist():
            if nodes["triCount"][x] == 0:
                c = int(nodes["leftFirst"][x])
                left[x], right[x], parent[c], parent[c + 1] = c, c + 1, x, x
                height[x] = 1 + max(height[c], height[c + 1])
    reach = np.concatenate(levels).tolist()
    leaves = [x for x in reach if left[x] < 0]
    if len(leaves) < 2:
        return nodes.copy(), idx.copy(), ic
    root = 0

    def path(y):   # -> ancestors of y, nearest first
        out = []
        while parent[y] >= 0:
            y = parent[y]
            out.append(y)
        return out

    def replace(q, old, new):
        if left[q] == old:
            left[q] = new
        else:
            right[q] = new

    def fix_heights(a):
        while a >= 0:
            height[a] = 1 + max(height[left[a]], height[right[a]])
            a = parent[a]

    def move(x, y):
        nonlocal root
        p = parent[x]
        s = right[p] if left[p] == x else left[p]
        g = parent[p]
        if g < 0:
            root, parent[s] = s, -1
        else:
            replace(g, p, s)
            parent[s] = g
        q = parent[y]
        if q < 0:
            root, parent[p] = p, -1
        else:
            replace(q, y, p)
            parent[p] = q
        left[p], right[p] = (x, y) if rng.random() < 0.5 else (y, x)
        parent[x] = parent[y] = p
        fix_heights(g)
        fix_heights(p)

    def try_move(x, y, limit):
        if x == root or y == parent[x] or y == x:
            return False
        anc = path(y)
        if x in anc:
            return False
        d = len(anc) - (parent[x] in anc)
        if d + 1 + max(height[x], height[y]) > limit:
            return False
        move(x, y)
        return True

    def dfs_sorted():
        order, stack = [], [root]
        while stack:
            a = stack.pop()
            if left[a] < 0:
                order.append(int(nodes["leftFirst"][a]))
            else:
                stack += [right[a], left[a]]
        return all(order[i] < order[i + 1] for i in range(len(order) - 1))

    done = tries = 0
    while (done < k or dfs_sorted()) and tries < 50 * k + 1000:
        tries += 1
        done += try_move(reach[rng.integers(len(reach))], reach[rng.integers(len(reach))], max_depth)
    while grow_to is not None and height[root] < grow_to:
        y = root
        while left[y] >= 0:
            y = left[y] if height[left[y]] >= height[right[y]] else right[y]
        try_move(leaves[rng.integers(len(leaves))], y, grow_to)
    return write_dfs(nodes, left, right, root), idx.copy(), ic


def shuffled_ranges(tree, seed, gap=0):
    """Family C: the leaf blocks placed in primIdx in a seeded order (never the DFS order), leftFirst updated.  gap > 0: 1 .. gap
    unreferenced entries holding triangle 0 after every block, so idxCount exceeds the referenced entries.  The source's tail of
    unreferenced entries (an SBVH's) is kept."""
    nodes, idx, ic = tree
    nodes = nodes.copy()
    leaves = dfs_leaves(nodes)
    rng = np.random.default_rng(seed)
    perm = rng.permutation(leaves.size)
    if leaves.size > 1 and (np.diff(perm) > 0).all():
        perm = np.roll(perm, 1)
    parts, pos = [], 0
    for j in perm.tolist():
        x = leaves[j]
        f, c = int(nodes["leftFirst"][x]), int(nodes["triCount"][x])
        parts.append(idx[f:f + c])
        nodes["leftFirst"][x] = pos
        pos += c
        if gap:
            g = int(rng.integers(1, gap + 1))
            parts.append(np.zeros(g, np.uint32))
            pos += g
    used = int(nodes["triCount"][leaves].sum())
    parts.append(np.zeros(ic - used, np.uint32))
    out = np.concatenate(parts).astype(np.uint32)
    return nodes, out, out.shape[0]


def renumbered(tree):
    """Family D's last step: sibling pairs numbered breadth-first (renumber_bfs)."""
    nodes, idx, ic = tree
    return renumber_bfs(nodes), idx.copy(), ic


FAMILIES = ["A0.3", "A1", "B", "C0", "C3", "DA", "DB", "DC"]


def family_tree(tree, fam, seed):
    """A tree of family `fam` (FAMILIES) made from a builder's tree: A0.3 / A1 swapped(0.3 / 1), B reinserted, C0 / C3
    shuffled_ranges(0 / 3), DA / DB / DC the BFS renumbering of swapped(0.3), reinserted and shuffled_ranges(3)."""
    if fam.startswith("D"):
        return renumbered(family_tree(tree, {"DA": "A0.3", "DB": "B", "DC": "C3"}[fam], seed))
    if fam.startswith("A"):
        return swapped(tree, seed, float(fam[1:]))
    if fam == "B":
        nodes = tree[0]
        return reinserted(tree, seed, max(4, min(400, nodes.shape[0] // 8)))
    return shuffled_ranges(tree, seed, int(fam[1:]))


def check_tree(tree, ntris):
    """The structural claims of every family: every node reachable exactly once (node 1 unused), leaf ranges disjoint and inside
    primIdx, children behind their parent, every primIdx entry a triangle, every interior box the fold of its children's.
    -> the tree's depth."""
    nodes, idx, ic = tree
    assert idx.shape[0] == ic and (idx < ntris).all()
    levels = tree_levels(nodes)
    reach = np.concatenate(levels)
    want = np.ones(nodes.shape[0], np.int64)
    want[1:2] = 0
    assert np.array_equal(np.bincount(reach, minlength=nodes.shape[0]), want), "every node but node 1 reachable exactly once"
    leaf = reach[nodes["triCount"][reach] > 0]
    inner = reach[nodes["triCount"][reach] == 0]
    c = nodes["leftFirst"][inner].astype(np.int64)
    assert (c > inner).all() and (c % 2 == 0).all(), "children sit behind their parent, in pairs from 2"
    f, n = nodes["leftFirst"][leaf].astype(np.int64), nodes["triCount"][leaf].astype(np.int64)
    o = np.argsort(f)
    assert (f + n <= ic).all() and (f[o][1:] >= (f + n)[o][:-1]).all(), "leaf ranges in bounds and disjoint"
    lmin, rmin, lmax, rmax = nodes["aabbMin"][c], nodes["aabbMin"][c + 1], nodes["aabbMax"][c], nodes["aabbMax"][c + 1]
    assert np.array_equal(bits_u32(nodes["aabbMin"][inner]), bits_u32(np.where(lmin < rmin, lmin, rmin)))
    assert np.array_equal(bits_u32(nodes["aabbMax"][inner]), bits_u32(np.where(lmax > rmax, lmax, rmax)))
    return len(levels) - 1


def small_scene(ntris=6000, seed=7):
    return scenes.procedural_scene(ntris, seed)


def ray_sets(verts, res=96, seed=0x123456):
    """primary (2 cameras) + shadow + diffuse rays over a scene; dict name -> RAY_DTYPE array (untraced)."""
    lo, hi = scenes.scene_bounds(verts)
    out = {}
    prim = []
    for kind in ("outside", "inside"):
        eye, view = R.bounds_camera(lo, hi, kind)
        prim.append(R.primary_rays(eye, view, res, res, 4))
    out["primary"] = np.concatenate(prim)
    return out, (lo, hi)


def derived_sets(traced_primary, verts, bounds):
    lo, hi = bounds
    eps = float((hi - lo).max() * 5e-7)
    light = (lo + hi) * 0.5 + np.array([0, (hi - lo)[1] * 0.45, 0], np.float32)
    return {"shadow": R.shadow_rays(traced_primary, light, eps), "diffuse": R.diffuse_rays(traced_primary, verts)}


def bits_u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


def nan_canonical(r):
    """A copy with every NaN t / u / v set to one pattern.  A hit with a NaN distance (Moeller-Trumbore overflowing on huge
    coordinates: 0 * inf) is accepted by the reference's `t < 0 || t > tmax` test; the NaN's bits are the floating-point unit's
    (0xffc00000 on x86, 0x7fffffff on the GPU), not the reference's."""
    r = r.copy()
    for f in ("t", "u", "v"):
        r[f][np.isnan(r[f])] = np.float32(np.nan)
    return r


def compare_hits(got, want):
    """-> dict of mismatch counts between two traced ray arrays (bit-exact fields)."""
    return {
        "prim": int((got["prim"] != want["prim"]).sum()),
        "t": int((bits_u32(got["t"]) != bits_u32(want["t"])).sum()),
        "u": int((bits_u32(got["u"]) != bits_u32(want["u"])).sum()),
        "v": int((bits_u32(got["v"]) != bits_u32(want["v"])).sum()),
    }


def classify_mismatches(got, want, verts):
    """Tie audit (SURVEY 8c): for rays whose prim differs from the oracle's, re-evaluate the engine's prim with the
    oracle's Moeller-Trumbore arithmetic.  exact-tie = bit-identical t; otherwise 'real'."""
    bad = np.nonzero(got["prim"] != want["prim"])[0]
    ties = real = 0
    v = verts.reshape(-1, 3, 4)
    for i in bad:
        p = int(got["prim"][i])
        ok, t, u, vv = portpy.tri_test(want["O"][i], want["D"][i], v[p, 0, :3], v[p, 1, :3], v[p, 2, :3], 1e30)
        if ok and np.float32(t).view(np.uint32) == want["t"][i].view(np.uint32):
            ties += 1
        else:
            real += 1
    return {"mismatch": int(bad.size), "tie_equivalent": ties, "real": real}


def random_transforms(count, seed, spread=60.0):
    """Row-major 4x4 instance transforms: rotation x (non-uniform) scale x translation, as tiny_bvh's bvhmat4 stores them."""
    rng = np.random.default_rng(seed)
    out = np.zeros((count, 16), np.float32)
    for i in range(count):
        a, b, c = rng.random(3) * 6.28
        rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
        ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
        rz = np.array([[np.cos(c), -np.sin(c), 0], [np.sin(c), np.cos(c), 0], [0, 0, 1]])
        m = np.eye(4)
        m[:3, :3] = (rx @ ry @ rz) @ np.diag(0.4 + rng.random(3) * 1.2)
        m[:3, 3] = (rng.random(3) - 0.5) * spread
        out[i] = m.astype(np.float32).reshape(-1)
    return out


# ---- input families away from the procedural atrium: signed zeros, power-of-two scales, large translations, long leaves
# Every family is seeded and deterministic.  The seeded scenes above all live in about [-40,40] x [0,30] x [-20,20] and hold no -0.

NEG_ZERO = np.float32(-0.0)


def signed_zero(v, mode, seed=0, frac=0.1):
    """Snap the coordinates nearest the floor plane y = 0 and the wall x = 0 (the `frac` of each closest to zero) to exact zeros.
    mode: "pos" all +0, "neg" all -0, "random" a seeded sign per vertex, "order" the sign triple of triangle t is the bit pattern of
    t % 8, so every vertex order of -0 and +0 occurs."""
    v = np.array(v, np.float32).reshape(-1, 4)
    rng = np.random.default_rng(seed)
    tri = np.arange(v.shape[0]) // 3
    for axis in (0, 1):
        a = np.abs(v[:, axis])
        snap = a <= np.quantile(a, frac)
        if mode == "pos":
            neg = np.zeros(v.shape[0], bool)
        elif mode == "neg":
            neg = np.ones(v.shape[0], bool)
        elif mode == "random":
            neg = rng.random(v.shape[0]) < 0.5
        elif mode == "order":
            neg = (((tri + axis) % 8) >> (np.arange(v.shape[0]) % 3)) & 1 == 1
        else:
            raise ValueError(mode)
        v[snap, axis] = np.where(neg[snap], NEG_ZERO, np.float32(0))
    return v


def count_neg_zero(a):
    a = np.ascontiguousarray(a, np.float32)
    return int(((a == 0) & np.signbit(a)).sum())


def zero_tri_cases():
    """The two orders of one triangle with a -0 and a +0 x-coordinate: BVH::Build's root aabbMin.x is the sign of the LAST one."""
    a = np.array([[NEG_ZERO, 0, 0, 0], [0, 1, 0, 0], [1, 0, 1, 0]], np.float32)
    b = a[[1, 0, 2]].copy()
    return a, b


def scaled(v, k):
    """Positions multiplied by exactly 2^k (float32 ldexp: subnormals round, as the scaled scene would)."""
    v = np.array(v, np.float32).reshape(-1, 4)
    v[:, :3] = np.ldexp(v[:, :3], k)
    return v


def scaled_rays(r, k):
    """Rays made at unit scale, moved to scale 2^k: O * 2^k, D and rD unchanged, t = 1e30."""
    r = r.copy()
    r["O"] = np.ldexp(r["O"], k)
    r["t"] = np.float32(1e30)
    return r


def translated(v, shift):
    """Positions plus `shift` in float32: far from the origin rounding merges vertices and makes zero-area triangles."""
    v = np.array(v, np.float32).reshape(-1, 4)
    v[:, :3] = v[:, :3] + np.float32(shift)
    return v


def snapped(v, q):
    """Positions rounded to multiples of 1 / q, with no -0 left (the + 0.0 turns -0 into +0).  Many fragment bounds then sit on
    the same planes, so BuildHQ's spatial splits often fail (every fragment on one side, tiny_bvh.h:2939), in big nodes too."""
    v = np.array(v, np.float32).reshape(-1, 4)
    q = np.float32(q)
    v[:, :3] = np.round(v[:, :3] * q) / q + np.float32(0.0)
    return v


def lattice_scene(n, seed, k=3):
    """n triangles whose vertices are seeded points of the integer lattice {0 .. k-1}^3: coincident, collinear and repeated
    vertices, and bounds on a few shared planes."""
    rng = np.random.default_rng(seed)
    v = np.zeros((n * 3, 4), np.float32)
    v[:, :3] = rng.integers(0, k, (n * 3, 3))
    return v


ONE_TRI = np.array([[0, 0, 0, 0], [1, 0, 0, 0], [0, 1, 0, 0]], np.float32)


def long_leaf_scene(name):
    """Trees whose CWBVH holds long chains of 3-triangle leaves (SplitLeafs of one big leaf):
    "identical": 700 identical triangles; "clusters": two clusters of 3,000 identical triangles 5 units apart;
    "collapsed": the 6,000-triangle scene at 2^40, where the SAH costs overflow and the tree collapses into a few huge leaves."""
    if name == "identical":
        return np.tile(ONE_TRI, (700, 1))
    if name == "clusters":
        a = np.tile(ONE_TRI, (3000, 1))
        b = a.copy()
        b[:, 0] += 5
        return np.concatenate([a, b])
    if name == "collapsed":
        return scaled(scenes.procedural_scene(6000, 7), 40)
    raise ValueError(name)


def cw_parents(nodes):
    """-> (parent of every wide node (-1 for the root and unreferenced records), inner-child count of every node) of bvh8Data."""
    n = np.ascontiguousarray(nodes).view(np.uint8).reshape(-1, 80)
    w = n.view(np.uint32).reshape(-1, 20)
    cnt = n.shape[0]
    ninner = ((n[:, 24:32] & 0x18) == 0x18).sum(1).astype(np.int64)
    parent = np.full(cnt, -1, np.int64)
    for x in range(cnt):
        for c in range(int(ninner[x])):
            if w[x, 4] + c < cnt:
                parent[w[x, 4] + c] = x
    return parent, ninner


def cw_depth_and_pending(nodes):
    """-> (depth of the wide tree, pending bound): the most ancestors with two or more inner children on a path from the root,
    the number of node groups the walk can hold at once."""
    parent, ninner = cw_parents(nodes)
    depth = pend = 0
    for x in range(parent.shape[0]):
        d = p = 0
        m = x
        while parent[m] >= 0:
            m = parent[m]
            d += 1
            p += int(ninner[m] >= 2)
        depth, pend = max(depth, d), max(pend, p)
    return depth, pend


def cw_exponents(nodes):
    """-> int8 [nodes, 3] exponent bytes of bvh8Data."""
    return np.ascontiguousarray(nodes).view(np.uint8).reshape(-1, 80)[:, 12:15].view(np.int8)


def cw_rd_limit(nodes):
    """The |rD| up to which a ray takes the CWBVH walk's integer slab test, from the bytes alone: 2^(127 - max(0, largest e)), or
    None when some e = -128 or some node origin |p| > 2^126."""
    e = cw_exponents(nodes).astype(np.int64)
    p = np.ascontiguousarray(nodes).view(np.float32).reshape(-1, 20)[:, :3]
    if (e == -128).any() or (np.abs(p) > np.float32(2.0 ** 126)).any():
        return None
    return np.float32(np.ldexp(1.0, 127 - max(0, int(e.max()))))


def octant_dirs():
    """The 8 direction octants as sign triples (+1 / -1), octant index = 4 * (x < 0) + 2 * (y < 0) + (z < 0)."""
    return np.array([[-1 if (o >> 2) & 1 else 1, -1 if (o >> 1) & 1 else 1, -1 if o & 1 else 1] for o in range(8)], np.float32)


def axis_rays(lo, hi, per_axis=16, seed=0):
    """Axis-aligned rays into a box, in all 8 octants: direction +-1 on one axis and zeros carrying the octant's sign on the
    others (rD = safercp(D), so +-1e30 there), origins outside the box on the travel axis, across the box and on its zero planes."""
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    ext = np.maximum(hi - lo, np.float32(1e-30))
    O, D = [], []
    for o, s in enumerate(octant_dirs()):
        for a in range(3):
            d = np.where(s < 0, NEG_ZERO, np.float32(0)).astype(np.float32)
            d[a] = s[a]
            for j in range(per_axis):
                p = (lo + ext * rng.random(3).astype(np.float32)).astype(np.float32)
                if j % 4 == 0:
                    p[(a + 1) % 3] = 0   # on a zero plane of the scene
                if j % 8 == 0:
                    p[(a + 2) % 3] = NEG_ZERO
                p[a] = lo[a] - ext[a] if s[a] > 0 else hi[a] + ext[a]
                O.append(p), D.append(d)
    r = R.make_rays(np.array(O), np.array(D), normalized=True)
    return r


def octant_rays(lo, hi, per_octant=64, seed=0):
    """Rays from points inside a box in random directions of every octant, per_octant each: the two test cameras never put a warp
    of rays into the octants with negative x and positive z."""
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    O, D = [], []
    for s in octant_dirs():
        O.append(lo + (hi - lo) * rng.random((per_octant, 3)).astype(np.float32))
        D.append(s * (np.float32(0.05) + rng.random((per_octant, 3)).astype(np.float32)))
    return R.make_rays(np.concatenate(O).astype(np.float32), np.concatenate(D).astype(np.float32))


def with_inf_rd(r):
    """The same rays with a user-supplied rD = 1 / D: +-inf on every zero direction component."""
    r = r.copy()
    with np.errstate(divide="ignore"):
        r["rD"] = (np.float32(1) / r["D"]).astype(np.float32)
    return r


def octant_blocks(r, seed=0):
    """Rays reordered into blocks of 32: blocks whose rays share one octant (every octant that occurs) alternating with blocks
    that mix octants, so every octant instance of the CWBVH walk and its per-lane form run."""
    oct_ = ((r["D"][:, 0] < 0) * 4 + (r["D"][:, 1] < 0) * 2 + (r["D"][:, 2] < 0)).astype(np.int64)
    rng = np.random.default_rng(seed)
    uni, mixed = [], []
    for o in range(8):
        idx = np.nonzero(oct_ == o)[0]
        full = idx.shape[0] // 32 * 32
        uni += [idx[k:k + 32] for k in range(0, full, 32)]
        mixed += list(idx[full:])
    mixed = np.array(mixed, np.int64)
    rng.shuffle(mixed)
    mixed = [mixed[k:k + 32] for k in range(0, mixed.shape[0], 32)]
    order = []
    for k in range(max(len(uni), len(mixed))):
        if k < len(uni):
            order.append(uni[k])
        if k < len(mixed):
            order.append(mixed[k])
    return r[np.concatenate(order)] if order else r


def rd_limit_rays(r, limit, seed=0):
    """Rays around the integer-slab-test bound: |rD.x| set to limit, the next float above it, 2 * limit - ulp, 2 * limit and inf
    (sign of D.x kept), in warps of their own and as one lane per warp of unchanged rays; plus origins at 2^126 and the next float."""
    rng = np.random.default_rng(seed)
    lim = np.float32(limit if limit is not None else 2.0 ** 127)
    with np.errstate(over="ignore"):
        two = np.float32(2) * lim   # inf when the bound is 2^127
    vals = [lim, np.nextafter(lim, np.float32(np.inf)), np.nextafter(two, np.float32(0)), two, np.float32(np.inf)]
    out = []
    for v in vals:
        for own in (True, False):
            s = r[rng.integers(0, r.shape[0], 64)].copy()
            sel = np.ones(64, bool) if own else (np.arange(64) % 32 == 7)
            sgn = np.where(s["D"][:, 0] < 0, np.float32(-1), np.float32(1))
            with np.errstate(over="ignore"):
                s["rD"][sel, 0] = (sgn[sel] * v).astype(np.float32)
            out.append(s)
    for o in (np.float32(2.0 ** 126), np.nextafter(np.float32(2.0 ** 126), np.float32(np.inf))):
        s = r[rng.integers(0, r.shape[0], 32)].copy()
        s["O"][:, 0] = -o
        out.append(s)
    return np.concatenate(out)


def shadow_at_hits(traced):
    """Shadow rays whose tmax is exactly the hit distance of a traced set (the any-hit test's t <= tmax edge)."""
    s = traced[traced["t"] < 1e30].copy()
    s["u"] = s["v"] = 0
    s["prim"] = 0
    return s
