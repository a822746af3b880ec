"""The host restatement of signed distances (tests/sdf_oracle.c, DESIGN.md §4.10), without a GPU: the per-triangle function with the
feature against orc_cp_triangle, each feature against its (u, v), and signs against an fp64 generalized winding number on closed meshes -
coplanar pairs, a sphere, a torus, a concave star, a hollow solid, two solids, a reversed mesh, vertex and edge bisectors, a 20-degree
wedge whose ridge defeats face normals, soups that differ in triangle order and corner rotation, and a cone with a 65,536-triangle fan."""
import numpy as np
import pytest

from tests import closest_oracle as co, sdf_oracle as so
from tests.test_closest_point import triangle_cases


# ---- closed meshes: (V (nv, 3) float64, F (nf, 3) int), outward by the right-hand rule on (v0, v1, v2) -----------------------------
def soup(V, F):
    """V[F] as float4 vertices, three per triangle"""
    t = np.asarray(V, np.float32)[np.asarray(F)].reshape(-1, 3)
    out = np.zeros((t.shape[0], 4), np.float32)
    out[:, :3] = t
    return out


def cube(lo=(-1, -1, -1), hi=(1, 1, 1)):
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    V = np.array([[(hi if (k >> a) & 1 else lo)[a] for a in range(3)] for k in range(8)])
    quads = [(0, 2, 3, 1), (4, 5, 7, 6), (0, 1, 5, 4), (2, 6, 7, 3), (0, 4, 6, 2), (1, 3, 7, 5)]
    F = [t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))]
    return V, np.array(F)


def icosphere(sub=2, r=1.0, c=(0, 0, 0)):
    t = (1 + 5 ** 0.5) / 2
    V = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    F = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
         (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    V = [np.array(v, np.float64) / np.linalg.norm(v) for v in V]
    for _ in range(sub):
        mid, G = {}, []

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = V[a] + V[b]
                V.append(p / np.linalg.norm(p))
                mid[k] = len(V) - 1
            return mid[k]
        for a, b, cc in F:
            ab, bc, ca = m(a, b), m(b, cc), m(cc, a)
            G += [(a, ab, ca), (b, bc, ab), (cc, ca, bc), (ab, bc, ca)]
        F = G
    return np.array(V) * r + np.asarray(c, np.float64), np.array(F)


def grid_surface(nu, nv, f):
    """a closed surface of quads over a periodic (u, v) grid: f(u, v) -> point"""
    U, W = np.meshgrid(np.arange(nu) / nu, np.arange(nv) / nv, indexing="ij")
    V = f(U.reshape(-1), W.reshape(-1))
    idx = lambda i, j: (i % nu) * nv + (j % nv)
    F = []
    for i in range(nu):
        for j in range(nv):
            a, b, c, d = idx(i, j), idx(i + 1, j), idx(i + 1, j + 1), idx(i, j + 1)
            F += [(a, b, c), (a, c, d)]
    return V, np.array(F)


def torus(R=1.0, r=0.35, nu=24, nv=12):
    def f(u, v):
        a, b = 2 * np.pi * u, 2 * np.pi * v
        return np.stack([(R + r * np.cos(b)) * np.cos(a), (R + r * np.cos(b)) * np.sin(a), r * np.sin(b)], 1)
    return oriented(*grid_surface(nu, nv, f))


def prism(poly, z0, z1, center=(0.0, 0.0)):
    """a polygon (star-shaped about `center`, counter-clockwise) extruded from z0 to z1; caps are fans from the centre"""
    n = len(poly)
    P = np.asarray(poly, np.float64)
    V = np.concatenate([np.c_[P, np.full(n, z0)], np.c_[P, np.full(n, z1)], [[*center, z0], [*center, z1]]])
    F = []
    for i in range(n):
        j = (i + 1) % n
        F += [(i, j, n + j), (i, n + j, n + i), (2 * n, j, i), (2 * n + 1, n + i, n + j)]
    return V, np.array(F)


def star(points=5, r0=0.4, r1=1.0):
    a = np.pi / 2 + np.arange(2 * points) * np.pi / points
    r = np.where(np.arange(2 * points) % 2 == 0, r1, r0)
    return oriented(*prism(np.c_[r * np.cos(a), r * np.sin(a)], -0.3, 0.3))


def volume(V, F):
    a, b, c = (V[F[:, k]] for k in range(3))
    return (a * np.cross(b, c)).sum() / 6


def oriented(V, F):
    return (V, F) if volume(V, F) > 0 else (V, F[:, ::-1].copy())


def join(*meshes):
    Vs, Fs, o = [], [], 0
    for V, F in meshes:
        Vs.append(V), Fs.append(F + o)
        o += V.shape[0]
    return np.concatenate(Vs), np.concatenate(Fs)


def hollow():
    """a sphere of radius 1 with a spherical cavity of radius 0.5: the inner shell faces the cavity"""
    V, F = icosphere(2, 0.5)
    return join(icosphere(3, 1.0), (V, F[:, ::-1].copy()))


def two_solids():
    return join(cube(), icosphere(2, 0.8, (3.0, 0.5, 0.2)))


def cone(fan=65536, r=1.0, h=2.0):
    """a cone whose apex is shared by `fan` triangles, closed by a base fan"""
    a = 2 * np.pi * np.arange(fan) / fan
    V = np.concatenate([np.c_[r * np.cos(a), r * np.sin(a), np.zeros(fan)], [[0, 0, h], [0, 0, 0]]])
    i = np.arange(fan)
    j = (i + 1) % fan
    F = np.concatenate([np.c_[i, j, np.full(fan, fan)], np.c_[j, i, np.full(fan, fan + 1)]])
    return V, F


def wedge(angle_deg=20.0, L=1.0, H=1.0):
    """a triangular prism whose ridge (the x = 0 edge along z) has the given dihedral angle; the two ridge faces are triangles 0-3, the
    +y face first, so the (d2, prim) tie at the ridge picks a +y triangle for points that lie on the -y side"""
    h = np.radians(angle_deg) / 2
    A, B, C = (0.0, 0.0), (-L * np.cos(h), L * np.sin(h)), (-L * np.cos(h), -L * np.sin(h))
    V = np.array([[*A, 0], [*B, 0], [*C, 0], [*A, H], [*B, H], [*C, H]], np.float64)
    F = np.array([(0, 3, 4), (0, 4, 1),       # +y face (A, B side)
                  (0, 2, 5), (0, 5, 3),       # -y face (A, C side)
                  (1, 4, 5), (1, 5, 2),       # back
                  (0, 1, 2), (3, 5, 4)])      # caps
    return oriented(V, F)


MESHES = {"cube": cube, "icosphere": lambda: icosphere(2), "torus": torus, "star": star, "hollow": hollow, "two_solids": two_solids,
          "wedge": wedge}


# ---- fp64 generalized winding number (Van Oosterom & Strackee solid angles) --------------------------------------------------------
def winding(V, F, P, chunk=64):
    tri = np.asarray(V, np.float64)[np.asarray(F)]
    out = np.zeros(P.shape[0])
    for s in range(0, P.shape[0], chunk):
        p = np.asarray(P[s: s + chunk], np.float64)[:, None, None, :]
        a, b, c = (tri[None, :, k, :] - p[:, :, 0, :] for k in range(3))
        la, lb, lc = (np.linalg.norm(x, axis=2) for x in (a, b, c))
        det = (a * np.cross(b, c)).sum(2)
        den = la * lb * lc + (a * b).sum(2) * lc + (b * c).sum(2) * la + (c * a).sum(2) * lb
        out[s: s + chunk] = 2 * np.arctan2(det, den).sum(1) / (4 * np.pi)
    return out


def sample_queries(V, F, rng, n=1500):
    """points around the mesh: uniform in a box 1.3 times its bounds, jittered surface points, and points along vertex and edge
    bisectors (angle-weighted normals in fp64) on both sides"""
    V = np.asarray(V, np.float64)
    lo, hi = V.min(0), V.max(0)
    ext = (hi - lo).max()
    c, half = (lo + hi) / 2, (hi - lo) / 2 * 1.3
    tri = V[F]
    k = rng.integers(0, F.shape[0], n)
    w = rng.dirichlet((1, 1, 1), n)
    onsurf = (tri[k] * w[:, :, None]).sum(1) + rng.normal(size=(n, 3)) * 0.02 * ext
    fn = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    fn /= np.maximum(np.linalg.norm(fn, axis=1, keepdims=True), 1e-300)
    vn = np.zeros_like(V)
    for j in range(3):
        e1, e2 = tri[:, (j + 1) % 3] - tri[:, j], tri[:, (j + 2) % 3] - tri[:, j]
        cosang = (e1 * e2).sum(1) / np.maximum(np.linalg.norm(e1, axis=1) * np.linalg.norm(e2, axis=1), 1e-300)
        np.add.at(vn, F[:, j], np.arccos(np.clip(cosang, -1, 1))[:, None] * fn)
    vn /= np.maximum(np.linalg.norm(vn, axis=1, keepdims=True), 1e-300)
    kv = rng.integers(0, V.shape[0], n // 2)
    t = rng.uniform(0.005, 0.08, (n // 2, 1)) * ext * rng.choice([-1, 1], (n // 2, 1))
    along_v = V[kv] + t * vn[kv]
    ke, ej = rng.integers(0, F.shape[0], n // 2), rng.integers(0, 3, n // 2)
    a, b = tri[ke, ej], tri[ke, (ej + 1) % 3]
    along_e = (a + b) / 2 + t * fn[ke]
    uni = c + rng.uniform(-1, 1, (n, 3)) * half
    return np.concatenate([uni, onsurf, along_v, along_e])


def qrows(P, r=np.inf):
    q = np.zeros((P.shape[0], 4), np.float32)
    q[:, :3] = P
    q[:, 3] = r
    return q


def check_signs(V, F, P, label, flip=False):
    """the oracle's signs equal the winding number's at every query farther than 1e-3 of the extent from the surface; -> records"""
    v = soup(V, F)
    q = qrows(P)
    rec = so.signed(v, q)
    assert (rec.view(np.uint32)[:, 3] != so.NO_PRIM).all()
    ext = np.ptp(np.asarray(V, np.float64), 0).max()
    far = np.abs(rec[:, 0]) > 1e-3 * ext
    inside = np.abs(winding(V, F, q[:, :3].astype(np.float64))) > 0.5
    neg = np.signbit(rec[:, 0])
    want = ~inside if flip else inside
    bad = far & (neg != want)
    assert not bad.any(), f"{label}: {int(bad.sum())} of {int(far.sum())} signs differ from the winding number, first {q[bad][:3]}"
    assert far.sum() > 0.8 * q.shape[0]
    return rec


# ---- tests ----------------------------------------------------------------------------------------------------------------------
def test_feature_function_matches_closest_point_bits():
    """(d2, u, v) of the feature form equal orc_cp_triangle's bit for bit on random and degenerate triangles, and every feature agrees
    with its (u, v)"""
    seen = set()
    for A, e1, e2, P, label in triangle_cases():
        d2, u, v = co.triangles(P, A, e1, e2)
        s2, su, sv, f = so.triangles(P, A, e1, e2)
        for x, y in ((d2, s2), (u, su), (v, sv)):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), label
        assert (f <= so.BC).all(), label
        for feat, ok in ((so.V0, (u == 0) & (v == 0)), (so.V1, (u == 1) & (v == 0)), (so.V2, (u == 0) & (v == 1)),
                         (so.AB, v == 0), (so.AC, u == 0), (so.FACE, (u > 0) & (v > 0))):
            sel = f == feat
            assert ok[sel].all(), f"{label}: feature {feat} with (u, v) {np.c_[u, v][sel & ~ok][:3]}"
        seen |= set(np.unique(f).tolist())
    assert seen == set(range(7)), seen


@pytest.mark.parametrize("name", sorted(MESHES))
def test_signs_match_winding_number(name):
    V, F = MESHES[name]()
    check_signs(V, F, sample_queries(V, F, np.random.default_rng(len(name))), name)


def test_reversed_mesh_flips_every_sign():
    V, F = icosphere(2)
    P = sample_queries(V, F, np.random.default_rng(3))
    a = check_signs(V, F, P, "icosphere")
    b = check_signs(V, F[:, ::-1].copy(), P, "reversed", flip=True)
    ext = 2.0
    far = np.abs(a[:, 0]) > 1e-3 * ext
    assert np.array_equal(np.signbit(a[far, 0]), ~np.signbit(b[far, 0]))
    assert np.allclose(np.abs(a[:, 0]), np.abs(b[:, 0]), rtol=1e-5, atol=1e-6)  # v0 differs, so the last bits may


def wedge_ridge_queries(V, rng, n=600):
    """points outside the ridge of wedge(): in the plane across the ridge, at 15-75 degrees from the bisector towards -y"""
    z = rng.uniform(0.2, 0.8, n) * V[:, 2].max()
    th = np.radians(rng.uniform(-75, -15, n))
    t = rng.uniform(0.02, 0.1, n)
    return np.c_[t * np.cos(th), t * np.sin(th), z]


def test_sharp_wedge_needs_edge_pseudonormals():
    """at a 20-degree ridge the tie picks the +y triangle for points on the -y side: its face normal gives the wrong sign there, the
    edge pseudonormal the right one"""
    V, F = wedge(20.0)
    P = wedge_ridge_queries(V, np.random.default_rng(7))
    rec = check_signs(V, F, P, "wedge ridge")
    assert not np.signbit(rec[:, 0]).any()
    table = so.prepare(soup(V, F))
    prim = rec.view(np.uint32)[:, 3]
    tri = soup(V, F).reshape(-1, 3, 4)[:, :, :3].astype(np.float32)
    c = tri[prim, 0] + rec[:, 1:2] * (tri[prim, 1] - tri[prim, 0]) + rec[:, 2:3] * (tri[prim, 2] - tri[prim, 0])
    face_sign = ((P - c) * table[prim, 0, :3]).sum(1)
    assert (face_sign < 0).sum() > 0.2 * P.shape[0], "the wedge does not defeat a face-normal sign"


def test_soup_order_and_rotation_keep_signs():
    """the same solid with triangles shuffled and corners rotated gets the same signs away from the surface"""
    rng = np.random.default_rng(9)
    for V, F in (star(), torus()):
        P = sample_queries(V, F, rng, n=600)
        base = check_signs(V, F, P, "base")
        perm = rng.permutation(F.shape[0])
        rot = rng.integers(0, 3, F.shape[0])
        G = np.stack([F[perm][np.arange(F.shape[0]), (rot + k) % 3] for k in range(3)], 1)
        other = check_signs(V, G, P, "shuffled+rotated")
        ext = np.ptp(V, 0).max()
        far = np.abs(base[:, 0]) > 1e-3 * ext
        assert np.array_equal(np.signbit(base[far, 0]), np.signbit(other[far, 0]))
        assert np.allclose(np.abs(base[:, 0]), np.abs(other[:, 0]), rtol=1e-5, atol=1e-6)


def test_welding_by_value():
    """-0 welds to +0, a NaN corner welds to nothing and its triangle adds zero normals; an indexed mesh's V[I] soup is the mesh"""
    V, F = cube()
    v = soup(V, F)
    t0 = so.prepare(v)
    z = v.copy()
    z[:, :3] = np.where(z[:, :3] == 0, np.float32(-0.0), z[:, :3])
    assert np.array_equal(so.prepare(z).view(np.uint32), t0.view(np.uint32))
    V2, F2 = icosphere(1)
    v2 = soup(V2, F2)
    t = so.prepare(v2)
    # each vertex pseudonormal of a corner equals that of every corner at the same position
    pos = v2[:, :3].view(np.uint32).reshape(-1, 3)
    vp = t[:, 1:4, :3].reshape(-1, 3)
    _, inv = np.unique(pos, axis=0, return_inverse=True)
    for g in range(inv.max() + 1):
        assert (vp[inv.reshape(-1) == g] == vp[inv.reshape(-1) == g][0]).all()
    bad = v2.copy()
    bad[4, 1] = np.nan
    tb = so.prepare(bad)
    # its face normal, the NaN corner's vertex (corner 1) and the two edges through it (AB, BC) are 0; its AC edge welds to the neighbour
    for slot in (0, 2, 4, 6):
        assert (tb[1, slot] == 0).all(), f"slot {slot} of the triangle with a NaN corner"
    assert (tb[1, 5, :3] != 0).any()
    assert np.isfinite(tb).all()


def test_large_fan_cone():
    """a cone with 65,536 triangles around its apex: signs along the axis above and below the apex, and around the cone"""
    V, F = cone()
    rng = np.random.default_rng(4)
    axis = np.c_[np.zeros(64), np.zeros(64), 2.0 + np.r_[rng.uniform(0.01, 0.3, 32), -rng.uniform(0.05, 1.5, 32)]]
    P = np.concatenate([axis, rng.uniform(-1.3, 1.3, (96, 3)) + [0, 0, 1]])
    rec = check_signs(V, F, P, "cone", )
    assert np.array_equal(np.signbit(rec[:64, 0]), np.r_[np.zeros(32, bool), np.ones(32, bool)])
