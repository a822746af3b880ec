"""A host model of engine handles across sequences of calls (include/tinybvh_b200.h).

Each Model holds what a handle holds, as the host restatements give it: the vertex soup (and the (V, I) of an indexed build that kept its
indices), the BVH2 (`tree`: nodes, primIdx padded to idx_count, the soup), the resident layouts, the BVH_GPU nodes, the CWBVH and the BVH2
its 8-wide collapse was taken from, `refittable`, whether a signed-distance or winding-number table is valid, and a generation that
changes exactly when the engine's does (a TLAS over the handle goes stale).  A TLAS model holds its instance records and the BLAS models
with the generations they had at build time.

Every transition is one call of the C-ABI restated: it returns the code the header documents and, when that is a refusal, leaves every
model as it was.  No transition computes anything itself: trees come from util.oracle_tree, ploc_oracle, optimize_oracle, PortBVH.refit,
to_bvh_gpu, PortCWBVH and cwbvh_refit_oracle.RefitCWBVH; walks from PortBVH / PortCWBVH / PortTLAS / PortTLASCW."""
import itertools

import numpy as np

from oracle import portpy
from tinybvh_b200 import _lib
from tests import ploc_oracle, util
from tests.cwbvh_refit_oracle import RefitCWBVH

OK, ARG, STATE, UNSUPPORTED = _lib.OK, _lib.E_ARG, _lib.E_STATE, _lib.E_UNSUPPORTED
BVH, GPU, CW = _lib.LAYOUT_BVH, _lib.LAYOUT_BVH_GPU, _lib.LAYOUT_CWBVH
BUILDERS = ("Build", "BuildAVX", "BuildHQ", "BuildPLOC")
FLAVOUR = {"Build": _lib.BUILD_REFERENCE, "BuildAVX": _lib.BUILD_AVX, "BuildHQ": _lib.BUILD_HQ, "BuildPLOC": _lib.BUILD_PLOC}
_generation = itertools.count(1)


def gather(V, I):
    """the soup V[I] of an indexed mesh, float4 rows with w = 0: what an indexed build and an indexed refit hold"""
    out = np.zeros((I.shape[0], 4), np.float32)
    out[:, :3] = np.asarray(V, np.float32).reshape(-1, 4)[I, :3]
    return out


def tree_of(builder, soup):
    """the BVH2 a builder leaves over a soup -> (PortBVH with primIdx padded to idxCount, referenced primIdx entries)"""
    if builder == "BuildPLOC":
        nodes, idx, _, _ = ploc_oracle.build(soup)
        return portpy.PortBVH(soup, nodes=nodes, prim_idx=idx), idx.shape[0]
    o = util.oracle_tree(soup, {"Build": 0, "BuildAVX": 1, "BuildHQ": 2}[builder])
    ic = int(getattr(o, "idx_count", o.prim_idx.shape[0]))
    idx = np.zeros(ic, np.uint32)
    idx[: o.prim_idx.shape[0]] = o.prim_idx
    return portpy.PortBVH(soup, nodes=np.asarray(o.nodes).view(portpy.NODE32).copy(), prim_idx=idx), o.prim_idx.shape[0]


class Model:
    def __init__(self, name):
        self.name, self.alive = name, True
        self.clear()

    def clear(self):
        """free_layouts: an empty handle"""
        self.kind = "empty"          # "blas" or "tlas"
        self.verts = None            # the soup the handle holds
        self.V = self.I = None       # the vertices and indices an indexed refittable build kept
        self.tree = None             # PortBVH: nodes, primIdx[idx_count], verts
        self.used_idx = 0            # primIdx entries the leaves reference (an SBVH's tail is unspecified)
        self.layouts = frozenset()
        self.gpu = None              # BVH_GPU nodes
        self.cw = None               # .nodes / .tris of the CWBVH
        self.cw_built = None         # the BVH2 nodes the kept collapse came from (None: no collapse kept)
        self.refittable = True
        self.pairs = False           # a BVH_GPU upload: walked through the child pairs derived from it
        self.sdf = self.wn = False
        self.inst = self.links = None
        self.tlas_layouts = frozenset()
        self.renew()

    def renew(self):
        self.gen = next(_generation)

    def snapshot(self):
        """everything a refusal must leave as it was"""
        return {k: v for k, v in self.__dict__.items()}

    def restore(self, s):
        self.__dict__.update(s)

    # ---- what the handle reports
    @property
    def has_tree(self):
        return self.tree is not None

    @property
    def idx_count(self):
        return 0 if self.tree is None else self.tree.prim_idx.shape[0]

    @property
    def cw_refs(self):
        """bvh8Tris records the wide leaves reference"""
        return 3 * int(self.tree.nodes["triCount"].sum()) if self.cw is not None else 0

    def info(self):
        """-> the tbvh_info fields the model fixes"""
        if self.tree is None:
            return dict(layouts=0, used_nodes=0, idx_count=0, max_depth=0, used_nodes_gpu=0, used_blocks=0, cwbvh_tri_count=0)
        return dict(layouts=sum(1 << l for l in self.layouts), used_nodes=0 if self.pairs else self.tree.nodes.shape[0],
                    idx_count=self.idx_count, max_depth=util.tree_depth(self.tree.nodes),
                    used_nodes_gpu=0 if self.gpu is None else self.gpu.shape[0],
                    used_blocks=0 if self.cw is None else self.cw.nodes.shape[0], cwbvh_tri_count=0 if self.cw is None else self.idx_count)

    def stale(self):
        """a TLAS: some BLAS was destroyed or its generation changed since the build"""
        return any(not b.alive or b.gen != g for b, g, _ in self.links)

    def tlas_walk_code(self, layout):
        want = CW if layout == CW else BVH
        if want not in self.tlas_layouts or self.stale():
            return STATE
        return OK

    def tlas_oracle(self, layout):
        """the two-level walk over the instance records of the build and every BLAS's current arrays (a refit that renews no generation
        rewrites them in place)"""
        if layout == CW:
            return portpy.PortTLASCW(self.tree.nodes, self.tree.prim_idx, self.inst, [b.cw for b, _, _ in self.links])
        return portpy.PortTLAS(self.tree.nodes, self.tree.prim_idx, self.inst, [b.tree for b, _, _ in self.links])


# ---- transitions: each takes the models of its handles and returns the expected code ---------------------------------------------

def build(m, builder, soup=None, V=None, I=None):
    """tbvh_build_flavour / tbvh_build_indexed"""
    if V is not None:
        soup = gather(V, I)
    tree, used = tree_of(builder, soup)
    m.clear()
    m.kind, m.verts, m.tree, m.used_idx, m.layouts = "blas", soup, tree, used, frozenset({BVH})
    m.refittable = builder != "BuildHQ"
    if V is not None and m.refittable:
        m.V, m.I = np.asarray(V, np.float32).reshape(-1, 4).copy(), np.asarray(I, np.uint32).copy()
    return OK


def build_batch(ms, builder, soups, VI=None):
    """tbvh_build_batch / tbvh_build_batch_hq: each handle as its own build leaves it.  The same handle twice is refused."""
    if len({id(m) for m in ms}) != len(ms):
        return ARG
    for k, m in enumerate(ms):
        if VI is not None and VI[k] is not None:
            build(m, builder, V=VI[k][0], I=VI[k][1])
        else:
            build(m, builder, soups[k])
    return OK


def upload_bvh(m, nodes, idx, soup):
    m.clear()
    m.kind, m.verts, m.layouts = "blas", soup, frozenset({BVH})
    m.tree, m.used_idx = portpy.PortBVH(soup, nodes=nodes, prim_idx=idx), idx.shape[0]
    return OK


def upload_bvh_gpu(m, gpu_nodes, src, soup):
    """src: the BVH2 the nodes were converted from, whose walks and queries the derived child pairs give"""
    m.clear()
    m.kind, m.verts, m.layouts, m.pairs, m.gpu = "blas", soup, frozenset({GPU}), True, gpu_nodes
    m.tree, m.used_idx = portpy.PortBVH(soup, nodes=src.nodes, prim_idx=src.prim_idx), src.prim_idx.shape[0]
    return OK


def convert_gpu(m):
    if BVH not in m.layouts:
        return STATE
    m.gpu = m.tree.to_bvh_gpu()
    m.layouts = m.layouts | {GPU}
    return OK


def convert_cw(ms):
    """tbvh_convert( CWBVH ) is ms of one; tbvh_convert_batch the rest"""
    if len({id(m) for m in ms}) != len(ms):
        return ARG
    if any(BVH not in m.layouts or m.kind == "tlas" for m in ms):
        return STATE
    for m in ms:
        if m.cw is not None:
            m.renew()      # drop_cwbvh: a TLAS may hold the old arrays
        t = m.tree
        m.cw = portpy.PortCWBVH(t.nodes, t.prim_idx[: m.used_idx], t.verts, idx_count=m.idx_count)
        m.cw_built = t.nodes.copy() if m.refittable else None
        m.layouts = m.layouts | {CW}
    return OK


def refit(ms, frames, keep, indexed=False):
    """tbvh_refit / tbvh_refit_layouts (ms of one) and tbvh_refit_batch / tbvh_refit_batch_indexed.  frames[k]: ("soup", the new soup) or,
    for tbvh_refit_batch_indexed, ("V", the new positions of the vertices the handle's kept indices read)."""
    if len({id(m) for m in ms}) != len(ms):
        return ARG
    for m, (kind, f) in zip(ms, frames):
        if kind == "V" and not indexed:
            return ARG
        if BVH not in m.layouts or m.pairs or not m.refittable:
            return STATE
        if keep and CW in m.layouts and m.cw_built is None:
            return STATE
        if kind == "soup" and f.shape[0] != m.verts.shape[0]:
            return ARG
        if kind == "V" and m.V is None:
            return STATE
        if kind == "V" and f.shape[0] != m.V.shape[0]:
            return ARG
    for m, (kind, f) in zip(ms, frames):
        f = np.ascontiguousarray(f, np.float32).copy()
        if kind == "V":
            m.V, soup = f, gather(f, m.I)
        else:
            soup = f
        if keep or m.cw is not None:
            m.renew()      # refit_trees: a TLAS holds the old root box; drop_cwbvh: the old arrays
        m.sdf = m.wn = False
        m.tree.refit(soup)
        m.verts = soup
        if keep:
            if GPU in m.layouts:
                m.gpu = m.tree.to_bvh_gpu()
            if CW in m.layouts:
                m.cw = RefitCWBVH(m.cw_built, m.tree.nodes, m.tree.prim_idx[: m.used_idx], soup, idx_count=m.idx_count)
        else:
            m.gpu = m.cw = m.cw_built = None
            m.layouts = frozenset({BVH})
    return OK


def optimize(m, max_rounds):
    """tbvh_optimize -> (code, rounds kept)"""
    from tests import optimize_oracle
    if m.kind == "tlas" or BVH not in m.layouts:
        return STATE, 0
    nodes, rounds, _, _ = optimize_oracle.optimize(m.tree.nodes, m.tree.prim_idx, max_rounds)
    if rounds == 0:
        return OK, 0
    m.tree = portpy.PortBVH(m.verts, nodes=nodes, prim_idx=m.tree.prim_idx)
    m.renew()
    m.gpu = m.cw = m.cw_built = None
    m.layouts = frozenset({BVH})
    m.sdf = m.wn = False
    return OK, rounds


def prepare(m, table):
    """tbvh_signed_distance_prepare (table "sdf") / tbvh_winding_number_prepare ("wn")"""
    if m.kind == "tlas":
        return UNSUPPORTED
    if m.tree is None:
        return STATE
    setattr(m, table, True)
    return OK


def query_code(m, table):
    """the code of a signed-distance (table "sdf") or winding-number ("wn") query"""
    if m.kind == "tlas":
        return UNSUPPORTED
    if m.tree is None or not getattr(m, table):
        return STATE
    return OK


def tlas_build(t, inst, blasses):
    """TLAS.Build / TLAS.Rebuild (tbvh_build_tlas / tbvh_build_tlas_update) over BLAS models; inst: raw records, Update()d here on a copy
    -> code; the model keeps the updated records"""
    if any(b is t or b.kind != "blas" for b in blasses):
        return STATE if all(b is not t for b in blasses) else ARG
    inst = inst.copy()
    lo = np.stack([b.tree.nodes[0]["aabbMin"] for b in blasses])[inst["blasIdx"]]
    hi = np.stack([b.tree.nodes[0]["aabbMax"] for b in blasses])[inst["blasIdx"]]
    portpy.instance_update(inst, lo, hi)
    fake = np.zeros((inst.shape[0] * 3, 4), np.float32)
    fake[0::3, :3], fake[1::3, :3], fake[2::3, :3] = inst["aabbMin"], inst["aabbMax"], inst["aabbMin"]
    tree = portpy.PortBVH(fake)
    t.clear()
    t.kind, t.tree, t.used_idx, t.layouts, t.refittable, t.verts = "tlas", tree, tree.prim_idx.shape[0], frozenset({BVH}), False, fake
    t.inst, t.links = inst, [(b, b.gen, None) for b in blasses]
    lay = {BVH, CW}
    for b in blasses:
        lay &= ({BVH} if BVH in b.layouts else set()) | ({CW} if CW in b.layouts else set())
    t.tlas_layouts = frozenset(lay)
    return OK


def destroy(m):
    m.alive = False
    return OK


def transition(fn, models, *args, **kw):
    """run a transition; a refusal restores every model it was given"""
    saved = [(m, m.snapshot()) for m in models]
    out = fn(*args, **kw)
    code = out[0] if isinstance(out, tuple) else out
    if code != OK:
        for m, s in saved:
            m.restore(s)
    return out


# ---- a pool of handles and the sequences run over it -------------------------------------------------------------------------------

def moved(v, seed, amp=0.03):
    """the same rows, every vertex displaced a little (an animation frame); w stays"""
    rng = np.random.default_rng(seed)
    w = np.array(v, np.float32, copy=True)
    ext = float((w[:, :3].max(0) - w[:, :3].min(0)).max())
    w[:, :3] += (rng.random((w.shape[0], 3), np.float32) - 0.5) * np.float32(amp * ext)
    return w


def pool_meshes():
    """-> per slot (soup, (V, I) or None): two procedural scenes, a closed icosphere inside the first (signs mean something), and an
    indexed icosphere beside it"""
    from tinybvh_b200 import scenes
    from tests.test_signed_distance import icosphere
    a = scenes.procedural_scene(2400, 131)
    lo, hi = scenes.scene_bounds(a)
    c, r = (lo + hi) * 0.5, float((hi - lo).max()) * 0.15
    V, F = icosphere(3, r, c)
    ball = np.zeros((F.size, 4), np.float32)
    ball[:, :3] = V.astype(np.float32)[F.reshape(-1)]
    V2, F2 = icosphere(2, r * 0.7, c + np.array([r * 1.5, 0, 0]))
    Vi = np.zeros((V2.shape[0], 4), np.float32)
    Vi[:, :3] = V2
    Ii = F2.astype(np.uint32).reshape(-1)
    return [(a, None), (ball, None), (gather(Vi, Ii), (Vi, Ii)), (scenes.procedural_scene(700, 132), None)]


class Pool:
    """Handles 0..3 over pool_meshes() and their models.  Every step applies a transition to the models; a subclass runs the same call on
    the engine (run) and compares (check).  self.log holds the steps so far, for a failure message."""
    N = 4

    def __init__(self):
        self.meshes = pool_meshes()
        self.models = [Model(k) for k in range(self.N)]
        self.log = []
        self.replica = None    # (slot, expected hits) of the last replicate

    def run(self, op, args, want):
        """the engine's call -> its code (the model alone: want)"""
        return want

    def check(self):
        pass

    def step(self, op, *args):
        self.log.append((op,) + args)
        ms, fn, margs = getattr(self, "_" + op)(*args)
        self.touched = [m for m in ms if m.alive]
        want = transition(fn, ms, *margs)
        got = self.run(op, args, want)
        assert got == want, f"{op}{args}: code {got}, the model says {want}\n" + self.trace()
        self.check()
        return want

    def trace(self):
        return "steps: " + " -> ".join(f"{s[0]}{s[1:]}" for s in self.log)

    # ---- the inputs of every operation, shared by the model and the engine
    def home(self, k):
        return self.meshes[k]

    def frame(self, k, seed, indexed):
        """the next animation frame of slot k: ("V", moved V) for an indexed refit of a handle that kept indices, else ("soup", moved soup)"""
        m = self.models[k]
        if indexed and m.V is not None:
            return "V", moved(m.V, seed)
        return "soup", moved(self.home(k)[0] if m.verts is None else m.verts, seed)

    def upload_source(self, k):
        return util.oracle_tree(self.home(k)[0], 0)

    def instances(self, blas_slots, seed):
        from tinybvh_b200 import api
        n = 6
        inst = np.zeros(n, api.BLAS_INSTANCE)
        inst["transform"] = util.random_transforms(n, seed, spread=30.0)
        inst["blasIdx"] = np.arange(n) % len(blas_slots)
        inst["mask"] = 0xFFFF
        return inst

    # ---- operations: -> (models touched, transition, its arguments)
    def _build(self, k, builder, indexed=False):
        soup, vi = self.home(k)
        if indexed and vi is not None:
            return [self.models[k]], build, (self.models[k], builder, None, vi[0], vi[1])
        return [self.models[k]], build, (self.models[k], builder, soup)

    def _build_batch(self, ks, builder):
        ms = [self.models[k] for k in ks]
        return ms, build_batch, (ms, builder, [self.home(k)[0] for k in ks], [self.home(k)[1] for k in ks])

    def _upload_bvh(self, k):
        o = self.upload_source(k)
        return [self.models[k]], upload_bvh, (self.models[k], o.nodes, o.prim_idx, self.home(k)[0])

    def _upload_bvh_gpu(self, k):
        o = self.upload_source(k)
        return [self.models[k]], upload_bvh_gpu, (self.models[k], o.to_bvh_gpu(), o, self.home(k)[0])

    def _convert_gpu(self, k):
        return [self.models[k]], convert_gpu, (self.models[k],)

    def _convert_cw(self, ks):
        ms = [self.models[k] for k in ks]
        return ms, convert_cw, (ms,)

    def _refit(self, ks, keep, indexed, seed, bad=None):
        """bad: "count" (one triangle short: TBVH_E_ARG) or "V" (new vertex rows for a handle that kept no indices: TBVH_E_STATE)"""
        frames = [self.frame(k, seed + k, indexed) for k in ks]
        if bad == "count":
            frames[0] = (frames[0][0], frames[0][1][:-3])
        if bad == "V":
            frames[0] = ("V", moved(self.home(2)[1][0], seed))
        ms = [self.models[k] for k in ks]
        self.frames = frames
        return ms, refit, (ms, frames, keep, indexed)

    def _optimize(self, k, rounds):
        return [self.models[k]], optimize, (self.models[k], rounds)

    def _prepare(self, k, table):
        return [self.models[k]], prepare, (self.models[k], table)

    def _tlas(self, k, blas_slots, seed, rebuild=False):
        self.inst = self.instances(blas_slots, seed)
        return [self.models[k]], tlas_build, (self.models[k], self.inst, [self.models[j] for j in blas_slots])

    def _destroy(self, k):
        old = self.models[k]
        self.models[k] = Model(k)
        return [old], destroy, (old,)

    def _replicate(self, k):
        m = self.models[k]
        if m.kind == "tlas":
            code = STATE if m.stale() or not m.tlas_layouts else OK
        else:
            code = OK if m.layouts & {BVH, CW} else STATE
        return [], lambda: code, ()


# ---- the sequences ---------------------------------------------------------------------------------------------------------------

def seq_reconvert_keeps_tables(p):
    """prepare both tables, then convert a handle that already holds a CWBVH again (single and batched): the tree and the vertices are
    unchanged, so the tables stay valid"""
    p.step("build", 1, "BuildAVX")
    p.step("convert_cw", [1])
    p.step("build", 0, "Build")
    p.step("convert_cw", [0])
    for k in (0, 1):
        p.step("prepare", k, "sdf")
        p.step("prepare", k, "wn")
    p.step("convert_cw", [1])
    p.step("convert_cw", [1, 0])
    p.step("convert_gpu", 1)


def seq_indexed(p):
    p.step("build", 2, "BuildAVX", True)
    p.step("optimize", 2, 3)
    p.step("refit", [2], 1, True, 10)
    p.step("refit", [2], 1, True, 11)
    p.step("convert_cw", [2])
    p.step("prepare", 2, "sdf")
    p.step("refit", [2, 0], 1, True, 12, "V")      # handle 0 is empty: refused before any handle is touched
    p.step("build", 0, "Build")
    p.step("refit", [0, 2], 1, True, 13)
    p.step("prepare", 2, "sdf")
    p.step("prepare", 2, "wn")


def seq_ploc_frames(p):
    p.step("build", 0, "BuildPLOC")
    p.step("convert_cw", [0])
    p.step("refit", [0], 1, False, 20)
    p.step("refit", [0], 1, False, 21)
    p.step("optimize", 0, 4)
    p.step("refit", [0], 1, False, 22)
    p.step("convert_cw", [0])
    p.step("build", 3, "Build")
    p.step("convert_cw", [3])
    p.step("tlas", 1, [0, 3], 23)
    p.step("replicate", 1)
    p.step("refit", [0, 3], 1, False, 24)
    p.step("tlas", 1, [0, 3], 23, True)
    p.step("replicate", 1)
    p.step("replicate", 1)


def seq_hq(p):
    p.step("build", 1, "BuildHQ")
    p.step("convert_cw", [1])
    p.step("refit", [1], 1, False, 30)
    p.step("refit", [1], 0, False, 31)
    p.step("optimize", 1, 4)
    p.step("refit", [1], 0, False, 32)
    p.step("prepare", 1, "sdf")
    p.step("prepare", 1, "wn")
    p.step("build", 0, "Build")


def seq_tlas_blas_swap(p):
    p.step("build", 0, "Build")
    p.step("build", 3, "BuildAVX")
    p.step("tlas", 1, [0, 3], 40)
    p.step("prepare", 1, "sdf")
    p.step("optimize", 1, 2)
    p.step("refit", [1], 0, False, 41)
    p.step("build", 1, "Build")                     # the TLAS handle rebuilt as a BLAS
    p.step("prepare", 1, "wn")
    p.step("tlas", 0, [1, 3], 42)                   # and a BLAS handle rebuilt as a TLAS: a TLAS over it goes stale
    p.step("tlas", 2, [0], 43)                      # a TLAS as a BLAS is refused


def seq_upload_pairs(p):
    p.step("upload_bvh_gpu", 0)
    p.step("prepare", 0, "sdf")
    p.step("prepare", 0, "wn")
    p.step("convert_cw", [0])
    p.step("refit", [0], 0, False, 50)
    p.step("build", 0, "Build")
    p.step("prepare", 0, "wn")
    p.step("upload_bvh", 0)


def seq_tlas_update(p):
    p.step("build", 0, "Build")
    p.step("build", 3, "Build")
    p.step("convert_cw", [0, 3])
    p.step("tlas", 1, [0, 3], 60)
    p.step("refit", [0], 1, False, 61)
    p.step("tlas", 1, [0, 3], 60, True)
    p.step("convert_cw", [3])
    p.step("tlas", 1, [0, 3], 60, True)
    p.step("refit", [3], 0, False, 62)              # no CWBVH is dropped: the TLAS stays valid in BVH layout over the refitted arrays
    p.step("destroy", 0)
    p.step("build", 0, "Build")
    p.step("tlas", 1, [0, 3], 63, True)


NAMED = {"reconvert_keeps_tables": seq_reconvert_keeps_tables, "indexed": seq_indexed, "ploc_frames": seq_ploc_frames, "hq": seq_hq,
         "tlas_blas_swap": seq_tlas_blas_swap, "upload_pairs": seq_upload_pairs, "tlas_update": seq_tlas_update}


def seq_random(p, seed, steps=12):
    """steps drawn from every transition over random handles; about one in eight is a call the engine refuses"""
    rng = np.random.default_rng(seed)
    p.step("build", int(rng.integers(4)), BUILDERS[int(rng.integers(4))])
    for s in range(steps - 1):
        k = int(rng.integers(4))
        m = p.models[k]
        blas = [j for j in range(4) if p.models[j].kind == "blas" and BVH in p.models[j].layouts and j != k]
        refuse = rng.random() < 0.125
        op = rng.choice(["build", "build_batch", "upload", "convert", "refit", "optimize", "prepare", "tlas", "destroy", "replicate"],
                        p=[0.14, 0.06, 0.06, 0.16, 0.2, 0.08, 0.14, 0.08, 0.03, 0.05])
        seed_s = seed * 100 + s
        if refuse:
            kind = int(rng.integers(4))
            if kind == 0 and m.kind == "blas" and BVH in m.layouts and m.refittable and not m.pairs:
                p.step("refit", [k], int(rng.integers(2)), False, seed_s, "count")
            elif kind == 1 and m.kind == "blas" and BVH in m.layouts and m.refittable and not m.pairs and m.V is None \
                    and not (CW in m.layouts and m.cw_built is None):
                p.step("refit", [k], int(rng.integers(2)), True, seed_s, "V")
            elif kind == 2:
                p.step("build_batch", [k, k], BUILDERS[int(rng.integers(4))])
            elif m.kind == "tlas":
                p.step("prepare", k, "sdf")
            else:
                p.step("convert_cw", [k, k])
            continue
        if op == "build":
            p.step("build", k, BUILDERS[int(rng.integers(4))], bool(rng.integers(2)))
        elif op == "build_batch":
            j = (k + 1 + int(rng.integers(3))) % 4
            p.step("build_batch", [k, j], BUILDERS[int(rng.integers(4))])
        elif op == "upload":
            p.step("upload_bvh_gpu" if rng.integers(2) else "upload_bvh", k)
        elif op == "convert":
            if rng.integers(3) == 0:
                p.step("convert_gpu", k)
            else:
                ks = [k] + ([blas[0]] if blas and rng.integers(2) else [])
                p.step("convert_cw", ks)
        elif op == "refit":
            ks = [k] + ([blas[-1]] if blas and rng.integers(2) else [])
            p.step("refit", ks, int(rng.integers(2)), bool(rng.integers(2)), seed_s)
        elif op == "optimize":
            p.step("optimize", k, int(rng.integers(1, 5)))
        elif op == "prepare":
            p.step("prepare", k, "sdf" if rng.integers(2) else "wn")
        elif op == "tlas" and blas:
            p.step("tlas", k, blas[: 1 + int(rng.integers(len(blas)))], seed_s, bool(rng.integers(2)))
        elif op == "destroy":
            p.step("destroy", k)
        elif op == "replicate" and m.kind == "blas" and (BVH in m.layouts or CW in m.layouts):
            p.step("replicate", k)
        else:
            p.step("prepare", k, "wn")


SEEDS = list(range(30))
