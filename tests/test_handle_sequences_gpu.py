"""Sequences of calls over a pool of four handles, each held to its host model (tests/handle_model.py) after every step: the return code;
info() and the download of every layout byte for byte (or TBVH_E_STATE); Intersect / IsOccluded in every layout bit for bit against the
model's walk; closest_point, sphere_overlap, signed_distance, winding_number at beta 2 and inf against the restatements (or the refusal of
a table that is not valid); overlap_pairs, nearest_triangles and distance_pairs for one pool pair and one self pair; a TLAS walked in
each BLAS layout (or TBVH_E_STATE when stale); a group replica walked as its source was when it was replicated.  The named sequences aim at
places where two features' bookkeeping meet; the seeded ones draw their steps at random, refusals included.  A failure prints the steps
so far."""
import ctypes as C

import numpy as np
import pytest

from tinybvh_b200 import _lib, api, rays as R, scenes
from tests import closest_oracle as co, handle_model as hm, meshdist_oracle as md, sdf_oracle as so, tritri_oracle as tt, util, wn_oracle as wo

pytestmark = pytest.mark.gpu
L = _lib.lib
NO_HITS = {"prim": 0, "t": 0, "u": 0, "v": 0}


def p(a):
    return C.c_void_p(a.ctypes.data)


def mesh_recs(arrays):
    """tbvh_mesh records of flat soups (vert_count 0) or ("V", rows) of indexed refits / (soup, (V, I)) of indexed builds"""
    recs = (_lib.Mesh * len(arrays))()
    for r, (v, vi) in zip(recs, arrays):
        if vi is None:
            r.verts, r.stride, r.vert_count, r.indices, r.prim_count = v.ctypes.data, 16, 0, None, v.shape[0] // 3
        else:
            r.verts, r.stride, r.vert_count, r.indices, r.prim_count = vi[0].ctypes.data, 16, vi[0].shape[0], vi[1].ctypes.data if vi[1] is not None else None, vi[2]
    return recs


class EnginePool(hm.Pool):
    def __init__(self):
        super().__init__()
        self.h = [api.BVH() for _ in range(self.N)]
        allv = np.concatenate([m[0] for m in self.meshes])
        sets, _ = util.ray_sets(allv, res=32)
        self.rays = sets["primary"]                                           # 2048 rays over the pool's meshes
        rng = np.random.default_rng(7)
        D = rng.normal(size=(2048, 3)).astype(np.float32) * 0.35 + np.array([0, 0, 1], np.float32)
        O = np.tile(np.array([[0, 0, -80]], np.float32), (D.shape[0], 1))
        self.tlas_rays = R.make_rays(O, D)                                     # toward the instances of Pool.instances
        lo, hi = scenes.scene_bounds(allv)
        self.q = np.zeros((600, 4), np.float32)
        self.q[:, :3] = (lo + (rng.random((600, 3)) * 1.2 - 0.1) * (hi - lo)).astype(np.float32)
        self.q[:, 3] = np.inf
        self.q_r = self.q.copy()
        self.q_r[:, 3] = np.float32(0.02 * float((hi - lo).max()))
        self.group = api.Group([0, 0]) if api.device_count() == 1 else api.Group()
        self.group_want = None

    # ---- the engine's calls
    def run(self, op, args, want):
        return getattr(self, "e_" + op)(*args)

    def e_build(self, k, builder, indexed=False):
        soup, vi = self.home(k)
        if indexed and vi is not None:
            V, I = vi
            return L().tbvh_build_indexed(self.h[k].h, p(V), 16, V.shape[0], p(I), I.shape[0] // 3, api.HOST, 1.0, 1.0, hm.FLAVOUR[builder])
        return L().tbvh_build_flavour(self.h[k].h, p(soup), 16, soup.shape[0] // 3, api.HOST, 1.0, 1.0, hm.FLAVOUR[builder])

    def e_build_batch(self, ks, builder):
        recs = mesh_recs([(self.home(k)[0], None if self.home(k)[1] is None else (self.home(k)[1][0], self.home(k)[1][1], self.home(k)[1][1].shape[0] // 3))
                          for k in ks])
        hs = (C.c_void_p * len(ks))(*[self.h[k].h.value for k in ks])
        if builder == "BuildHQ":
            return L().tbvh_build_batch_hq(hs, recs, len(ks), api.HOST, 1.0, 1.0)
        return L().tbvh_build_batch(hs, recs, len(ks), api.HOST, 1.0, 1.0, hm.FLAVOUR[builder])

    def e_upload_bvh(self, k):
        o, v = self.upload_source(k), self.home(k)[0]
        return L().tbvh_upload_bvh(self.h[k].h, p(o.nodes), o.nodes.shape[0], p(o.prim_idx), o.prim_idx.shape[0], p(v), 16, v.shape[0] // 3, api.HOST)

    def e_upload_bvh_gpu(self, k):
        o, v = self.upload_source(k), self.home(k)[0]
        g = o.to_bvh_gpu()
        return L().tbvh_upload_bvh_gpu(self.h[k].h, p(g), g.shape[0], p(o.prim_idx), o.prim_idx.shape[0], p(v), 16, v.shape[0] // 3, api.HOST)

    def e_convert_gpu(self, k):
        return L().tbvh_convert(self.h[k].h, api.LAYOUT_BVH_GPU)

    def e_convert_cw(self, ks):
        if len(ks) == 1:
            return L().tbvh_convert(self.h[ks[0]].h, api.LAYOUT_CWBVH)
        return L().tbvh_convert_batch((C.c_void_p * len(ks))(*[self.h[k].h.value for k in ks]), len(ks), api.LAYOUT_CWBVH)

    def e_refit(self, ks, keep, indexed, seed, bad=None):
        frames = self.frames
        if len(ks) == 1 and not indexed:
            f = frames[0][1]
            fn = L().tbvh_refit_layouts if keep else L().tbvh_refit
            return fn(self.h[ks[0]].h, p(f), 16, f.shape[0] // 3, api.HOST)
        arrays = []
        for k, (kind, f) in zip(ks, frames):
            n = self.h[k].info().prim_count
            arrays.append((f, None) if kind == "soup" else (f, (f, None, n)))
        recs = mesh_recs(arrays)
        hs = (C.c_void_p * len(ks))(*[self.h[k].h.value for k in ks])
        fn = L().tbvh_refit_batch_indexed if indexed else L().tbvh_refit_batch
        return fn(hs, recs, len(ks), api.HOST, int(keep))

    def e_optimize(self, k, rounds):
        r, s = C.c_uint32(), C.c_float()
        return L().tbvh_optimize(self.h[k].h, rounds, 1.0, 1.0, C.byref(r), C.byref(s)), int(r.value)

    def e_prepare(self, k, table):
        return (L().tbvh_signed_distance_prepare if table == "sdf" else L().tbvh_winding_number_prepare)(self.h[k].h)

    def e_tlas(self, k, blas_slots, seed, rebuild=False):
        inst = self.inst.copy()
        hs = (C.c_void_p * len(blas_slots))(*[self.h[j].h.value for j in blas_slots])
        if rebuild:
            return L().tbvh_build_tlas_update(self.h[k].h, p(inst), 192, inst.shape[0], api.HOST, hs, len(blas_slots), 1.0, 1.0)
        for i in range(inst.shape[0]):
            rc = L().tbvh_instance_update(C.c_void_p(inst[i:i + 1].ctypes.data), self.h[blas_slots[int(inst["blasIdx"][i])]].h)
            if rc != _lib.OK:
                return rc
        return L().tbvh_build_tlas(self.h[k].h, p(inst), 192, inst.shape[0], hs, len(blas_slots), 1.0, 1.0)

    def e_destroy(self, k):
        rc = L().tbvh_bvh_destroy(self.h[k].h)
        self.h[k].h = None
        self.h[k] = api.BVH()
        return rc

    def e_replicate(self, k):
        m = self.models[k]
        ms = C.c_double()
        rc = L().tbvh_group_replicate(self.group.h, self.h[k].h, C.byref(ms))
        if rc == _lib.OK:
            layout = api.LAYOUT_CWBVH if (hm.CW in (m.tlas_layouts if m.kind == "tlas" else m.layouts)) else api.LAYOUT_BVH
            rays = self.tlas_rays if m.kind == "tlas" else self.rays
            want = rays.copy()
            (m.tlas_oracle(layout) if m.kind == "tlas" else (m.cw if layout == api.LAYOUT_CWBVH else m.tree)).intersect(want)
            self.group_want = (layout, rays, want)
        return rc

    # ---- the checks after every step
    def check(self):
        for k, m in enumerate(self.models):
            self.check_handle(k, m)
        self.check_pairs()
        if self.group_want is not None:
            layout, rays, want = self.group_want
            got = rays.copy()
            api.check(L().tbvh_group_intersect(self.group.h, layout, p(got), 128, got.shape[0]))
            assert util.compare_hits(util.nan_canonical(got), util.nan_canonical(want)) == NO_HITS, "group replica\n" + self.trace()

    def fail(self, k, what):
        return f"handle {k}: {what}\n" + self.trace()

    def check_handle(self, k, m):
        b = self.h[k]
        i = b.info()
        want = m.info()
        got = {f: getattr(i, f) for f in want}
        assert got == want, self.fail(k, f"info {got} != model {want}")
        # downloads
        n32, idx = np.zeros(max(i.used_nodes, 1), api.NODE32), np.zeros(max(i.idx_count, 1), np.uint32)
        rc = L().tbvh_download_bvh(b.h, p(n32), p(idx), api.HOST)
        assert rc == (_lib.OK if hm.BVH in m.layouts else _lib.E_STATE), self.fail(k, f"download_bvh {rc}")
        if rc == _lib.OK:
            assert np.array_equal(n32.view(np.uint32), m.tree.nodes.view(np.uint32)), self.fail(k, "BVH nodes")
            assert np.array_equal(idx[: m.used_idx], m.tree.prim_idx[: m.used_idx]), self.fail(k, "primIdx")
        n64 = np.zeros(max(i.used_nodes_gpu, 1), api.NODE64)
        rc = L().tbvh_download_bvh_gpu(b.h, p(n64), api.HOST)
        assert rc == (_lib.OK if m.gpu is not None else _lib.E_STATE), self.fail(k, f"download_bvh_gpu {rc}")
        if rc == _lib.OK:
            assert np.array_equal(n64.view(np.uint32), np.ascontiguousarray(m.gpu).view(np.uint32)), self.fail(k, "BVH_GPU nodes")
        d8, t8 = np.zeros((max(i.used_blocks, 1), 4), np.float32), np.zeros((max(i.cwbvh_tri_count, 1) * 3, 4), np.float32)
        rc = L().tbvh_download_cwbvh(b.h, p(d8), p(t8), api.HOST)
        assert rc == (_lib.OK if m.cw is not None else _lib.E_STATE), self.fail(k, f"download_cwbvh {rc}")
        if rc == _lib.OK:
            assert np.array_equal(d8.view(np.uint32), m.cw.nodes.view(np.uint32)), self.fail(k, "bvh8Data")
            assert np.array_equal(t8[: m.cw_refs].view(np.uint32), m.cw.tris[: m.cw_refs].view(np.uint32)), self.fail(k, "bvh8Tris")
        # walks
        if m.kind == "tlas":
            for layout in (api.LAYOUT_BVH, api.LAYOUT_CWBVH):
                self.check_walk(k, layout, m.tlas_walk_code(layout), lambda: m.tlas_oracle(layout), self.tlas_rays, tlas=True)
            q = self.q[:4].copy()
            assert L().tbvh_closest_point(b.h, p(q), p(np.zeros((4, 4), np.float32)), 4, api.HOST, None) == _lib.E_UNSUPPORTED
            for table in ("sdf", "wn"):
                assert self.query(b, table, self.q[:4]) == (hm.query_code(m, table), None)
            return
        tree_code = _lib.OK if m.tree is not None else _lib.E_STATE
        for layout in (api.LAYOUT_BVH, api.LAYOUT_BVH_GPU):
            self.check_walk(k, layout, tree_code, lambda: m.tree, self.rays)
        self.check_walk(k, api.LAYOUT_CWBVH, _lib.OK if m.cw is not None else _lib.E_STATE, lambda: m.cw, self.rays, cw=True)
        if m.tree is None:
            return
        # proximity queries
        t, v = m.tree, m.verts
        got = np.zeros((self.q.shape[0], 4), np.float32)
        api.check(L().tbvh_closest_point(b.h, p(self.q), p(got), self.q.shape[0], api.HOST, None))
        assert np.array_equal(got.view(np.uint32), co.walk(t.nodes, t.prim_idx, v, self.q).view(np.uint32)), self.fail(k, "closest_point")
        words = np.zeros((self.q.shape[0] + 31) // 32, np.uint32)
        api.check(L().tbvh_sphere_overlap(b.h, p(self.q_r), p(words), self.q.shape[0], api.HOST, None))
        assert np.array_equal(words, co.walk(t.nodes, t.prim_idx, v, self.q_r, any_=True)), self.fail(k, "sphere_overlap")
        for table in ("sdf", "wn"):
            code, out = self.query(b, table, self.q)
            assert code == hm.query_code(m, table), self.fail(k, f"{table} query {code}, the model says {hm.query_code(m, table)}")
            if code != _lib.OK:
                continue
            if table == "sdf":
                want = so.brute(t.nodes, t.prim_idx, v, self.q, walk=True)
                assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), self.fail(k, "signed_distance")
            else:
                w = wo.Table(t.nodes, t.prim_idx, v)
                for beta, o in zip((2.0, np.inf), out):
                    assert np.array_equal(o.view(np.uint32), w.query(self.q, beta).view(np.uint32)), self.fail(k, f"winding_number beta {beta}")

    def query(self, b, table, q):
        q = np.ascontiguousarray(q)
        if table == "sdf":
            out = np.zeros((q.shape[0], 4), np.float32)
            rc = L().tbvh_signed_distance(b.h, p(q), p(out), q.shape[0], api.HOST, None)
            return rc, (out if rc == _lib.OK else None)
        outs = []
        for beta in (2.0, np.inf):
            out = np.zeros(q.shape[0], np.float32)
            rc = L().tbvh_winding_number(b.h, p(q), p(out), q.shape[0], beta, api.HOST, None)
            if rc != _lib.OK:
                return rc, None
            outs.append(out)
        return _lib.OK, outs

    def check_walk(self, k, layout, code, oracle, rays, cw=False, tlas=False):
        got = rays.copy()
        rc = L().tbvh_intersect(self.h[k].h, layout, p(got), 128, got.shape[0])
        assert rc == code, self.fail(k, f"Intersect in layout {layout}: {rc}, the model says {code}")
        bits = np.zeros((rays.shape[0] + 31) // 32, np.uint32)
        rc = L().tbvh_occluded(self.h[k].h, layout, p(rays), 128, rays.shape[0], p(bits))
        assert rc == code, self.fail(k, f"IsOccluded in layout {layout}: {rc}")
        if code != _lib.OK:
            return
        o = oracle()
        want = rays.copy()
        o.intersect(want)
        if tlas:
            assert np.array_equal(got.view(np.uint32).reshape(-1, 32)[:, 11:16], want.view(np.uint32).reshape(-1, 32)[:, 11:16]), self.fail(k, f"TLAS Intersect layout {layout}")
        else:
            assert util.compare_hits(util.nan_canonical(got), util.nan_canonical(want)) == NO_HITS, self.fail(k, f"Intersect layout {layout}")
        if cw:
            occ = np.packbits(want["t"] < rays["t"], bitorder="little").view(np.uint8)
            occ = np.pad(occ, (0, bits.nbytes - occ.nbytes)).view(np.uint32)
        else:
            occ = o.occluded(rays)
        assert np.array_equal(bits, occ), self.fail(k, f"IsOccluded layout {layout}")

    def check_pairs(self):
        """overlap_pairs / nearest_triangles / distance_pairs for the pool pair (0, 1) and handle 2 with itself, when they hold trees"""
        for a, c in ((0, 1), (2, 2)):
            ma, mc = self.models[a], self.models[c]
            if ma.kind != "blas" or mc.kind != "blas":
                continue
            A, B = self.h[a], self.h[c]
            va = None if a == c else ma.verts
            t = mc.tree
            pairs = A.overlap_pairs(None if a == c else B)
            assert np.array_equal(pairs, tt.tree(t.nodes, t.prim_idx, mc.verts, va)[0]), self.fail(a, f"overlap_pairs with {c}")
            d, j = A.nearest_triangles(None if a == c else B)
            wd, wj = md.nearest(t.nodes, t.prim_idx, mc.verts, va)
            assert np.array_equal(d.view(np.uint32), wd.view(np.uint32)) and np.array_equal(j, wj), self.fail(a, f"nearest_triangles with {c}")
            r = float(np.float32(0.01 * float(np.ptp(mc.verts[:, :3], 0).max())))
            got = A.distance_pairs(None if a == c else B, r)
            assert np.array_equal(got, md.pairs(t.nodes, t.prim_idx, mc.verts, va, r=r)[0]), self.fail(a, f"distance_pairs with {c}")


@pytest.fixture
def pool(gpu):
    p = EnginePool()
    yield p
    p.group.close()


@pytest.mark.parametrize("name", list(hm.NAMED))
def test_named(pool, name):
    hm.NAMED[name](pool)


@pytest.mark.parametrize("seed", hm.SEEDS)
def test_random(pool, seed):
    hm.seq_random(pool, seed)
