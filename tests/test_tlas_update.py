"""CPU side of tbvh_build_tlas_update: the prototype, the refusals that need no device, and the arithmetic the device kernel shares
with the host (tinybvh_b200/csrc/instance_update.cuh, reached here through tbvh_instance_update_box) on the inputs BLASInstance::Update is
sensitive to - a wrong contraction or fold shows here, before a GPU is involved."""
import ctypes as C
import itertools
import os
import re

import numpy as np

from oracle import portpy
from tinybvh_b200 import _lib, api

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NZ = np.float32(-0.0)


def update_families(seed=5):
    """name -> transforms [n, 16]: what Update's rounding, its `w != 1` test, its `det == 0` exit and its box fold depend on."""
    rng = np.random.default_rng(seed)
    fam = {}
    perm = []
    for p in itertools.permutations(range(3)):
        for signs in itertools.product((1.0, -1.0), repeat=3):
            m = np.zeros((4, 4), np.float32)
            for r in range(3):
                m[r, p[r]] = signs[r]
            m[3, 3] = 1
            perm.append(m.reshape(-1))
    perm = np.array(perm, np.float32)
    neg = perm.copy()
    neg[neg == 0] = NZ                                    # the zeros of the matrix negative: products are -0, sums decide the sign
    fam["permutation_mirror"] = np.concatenate([perm, neg])

    def affine(n, scale=1.0, shift=0.0):
        t = np.zeros((n, 4, 4), np.float32)
        t[:, :3, :3] = (rng.random((n, 3, 3), np.float32) - 0.5) * 2
        t[:, :3, 3] = (rng.random((n, 3), np.float32) - 0.5) * 10
        t[:, :3, :3] *= np.float32(scale)
        t[:, :3, 3] += np.float32(shift)
        t[:, 3, 3] = 1
        return t
    s = affine(40)
    s[:10, 1, :] = 0                                      # a zero row: every cofactor product through it is 0, det == 0
    s[10:20, :3, 2] = 0                                   # a zero column
    s[20:30, 2, :] = s[20:30, 0, :]                       # two equal rows
    s[30:, :, :] = 0                                      # the zero matrix
    fam["singular"] = s.reshape(-1, 16)
    pr = affine(40)
    pr[:20, 3, :3] = (rng.random((20, 3), np.float32) - 0.5) * 0.05
    pr[20:, 3, :3] = np.array([1, 0, 0], np.float32)      # w == 1 exactly where the corner's x is 0, another value elsewhere
    fam["projective"] = pr.reshape(-1, 16)
    fam["scale_2^-60"] = affine(30, scale=2.0 ** -60).reshape(-1, 16)
    fam["scale_2^60"] = affine(30, scale=2.0 ** 60).reshape(-1, 16)
    fam["translation_2^20"] = affine(30, shift=2.0 ** 20).reshape(-1, 16)
    return fam


ZERO_BOXES = [((NZ, -1.0, -2.0), (0.0, NZ, 3.0)), ((0.0, 0.0, 0.0), (NZ, NZ, NZ)), ((-1.0, NZ, 0.0), (1.0, 0.0, NZ)), ((-1.5, -0.7, -2.2), (1.1, 2.3, 0.9))]


def records(transforms, blas_idx=0):
    inst = np.zeros(transforms.shape[0], api.BLAS_INSTANCE)
    inst["transform"], inst["blasIdx"], inst["mask"] = transforms, blas_idx, 0xFFFF
    inst["dummy"] = 0xFEED0000 + np.arange(transforms.shape[0], dtype=np.uint32)[:, None]
    return inst


def test_shared_update_routine_matches_the_oracle_on_sensitive_inputs():
    L = _lib.lib()
    for name, T in update_families().items():
        for lo, hi in ZERO_BOXES:
            lo, hi = np.array(lo, np.float32), np.array(hi, np.float32)
            want, got = records(T), records(T)
            with np.errstate(all="ignore"):
                portpy.instance_update(want, lo, hi)
            for i in range(got.shape[0]):
                assert L.tbvh_instance_update_box(C.c_void_p(got[i:i + 1].ctypes.data), lo.ctypes.data_as(C.c_void_p), hi.ctypes.data_as(C.c_void_p)) == 0
            assert got.tobytes() == want.tobytes(), (name, lo, hi)
    # the families do reach the branches they are named for
    sing = records(update_families()["singular"])
    portpy.instance_update(sing, np.float32([-1, -1, -1]), np.float32([1, 1, 1]))
    assert np.isfinite(sing["invTransform"]).all(), "det == 0 stores the cofactors, not a division by zero"


def test_prototype_is_declared_and_bound():
    hdr = open(os.path.join(REPO, "include", "tinybvh_b200.h")).read()
    m = re.search(r"int tbvh_build_tlas_update\(([^;]*)\);", hdr)
    assert m and len(m.group(1).split(",")) == len(_lib.SYMBOLS["tbvh_build_tlas_update"][1]) == 9
    assert hasattr(_lib.lib(), "tbvh_build_tlas_update")


def test_argument_refusals_need_no_device():
    """NULL handles, zero counts, a short stride: refused with TBVH_E_ARG before any device call, as tbvh_build_tlas refuses them."""
    L = _lib.lib()
    inst = records(update_families()["projective"])
    fake = (C.c_void_p * 1)(None)
    p = C.c_void_p(inst.ctypes.data)
    before = inst.tobytes()
    assert L.tbvh_build_tlas_update(None, p, 192, 4, api.HOST, fake, 1, 1.0, 1.0) == _lib.E_ARG
    assert L.tbvh_build_tlas(None, p, 192, 4, fake, 1, 1.0, 1.0) == _lib.E_ARG
    assert inst.tobytes() == before
