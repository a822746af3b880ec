"""The Python layer of tbvh_mesh_toi / tbvh_mesh_toi_pairs (time_of_impact / impact_pairs): an end frame that is not 3 x triCount rows
of 3 or 4 floats, a missing other_end, or a self query given a second end frame is refused with TbvhError before any native call
(the C-ABI reads exactly 3 x prim_count rows, so a short frame would be read past its end), for numpy arrays and tensors, in host and
device space; frames of the right shape become float32 rows at stride 12 or 16."""
import ctypes as C

import numpy as np
import pytest

from tinybvh_b200 import api
from tinybvh_b200._lib import TbvhError


class Mesh(api.BVH):
    """a handle stand-in of n triangles that never reaches the device"""

    def __init__(self, n):
        self.n, self.device, self.h = n, 0, C.c_void_p()

    triCount = property(lambda s: s.n)


def frames(n):
    import torch
    return {
        "short": np.zeros((3 * n - 1, 4), np.float32),
        "long": np.zeros((3 * n + 3, 4), np.float32),
        "columns": np.zeros((3 * n, 5), np.float32),
        "flat": np.zeros(3 * n * 4, np.float32),
        "short tensor": torch.zeros((3 * n - 3, 3)),
        "per-triangle": np.zeros((n, 9), np.float32),
    }


@pytest.mark.parametrize("method", ["time_of_impact", "impact_pairs"])
@pytest.mark.parametrize("stream", [None, 7])
def test_frames_of_another_shape_are_refused(method, stream):
    a, b = Mesh(10), Mesh(4)
    good_a, good_b = np.zeros((30, 4), np.float32), np.zeros((12, 3), np.float32)
    call = lambda *args, **kw: getattr(a, method)(*args, xi=1e-3, stream=stream, **kw)  # noqa: E731
    for label, bad in frames(10).items():
        with pytest.raises(TbvhError, match="end must be"):
            call(bad)
        with pytest.raises(TbvhError, match="end must be"):
            call(bad, b, good_b)
    for label, bad in frames(4).items():
        with pytest.raises(TbvhError, match="other_end must be"):
            call(good_a, b, bad)
    with pytest.raises(TbvhError, match="other_end must be"):
        call(good_a, b, good_a)          # a's frame passed for b
    with pytest.raises(TbvhError, match="needs its end frame"):
        call(good_a, b)
    with pytest.raises(TbvhError, match="one end frame"):
        call(good_a, None, good_a.copy())
    with pytest.raises(TbvhError, match="one end frame"):
        call(good_a, a, good_a.copy())
    with pytest.raises(TbvhError, match="xi"):
        getattr(a, method)(good_a)


def test_frames_of_the_right_shape_become_float32_rows():
    import torch
    a, b = Mesh(10), Mesh(4)
    L, o, args, dev, keep = a._toi_args(np.zeros((30, 3), np.float64), b, torch.zeros((12, 4), dtype=torch.float64), 0.0, 1e-3, 8, None)
    assert o is b and dev is None
    assert [k.dtype for k in keep] == [np.float32, np.float32] and [k.shape for k in keep] == [(30, 3), (12, 4)]
    assert (args[2], args[5]) == (12, 16) and args[1].value == keep[0].ctypes.data and args[4].value == keep[1].ctypes.data
    e = np.zeros((30, 4), np.float32)
    L, o, args, dev, keep = a._toi_args(e, a, e, 0.0, 1e-3, 8, None)   # a self query may repeat end itself
    assert o is a and len(keep) == 1 and args[1].value == args[4].value and args[2] == args[5] == 16
