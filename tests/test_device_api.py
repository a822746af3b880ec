"""CPU-side checks of the device API: the public device header compiles on its own, and the ctypes mirror of tbvh_view has the C
struct's layout."""
import ctypes as C
import os
import subprocess
import tempfile

import pytest

from tinybvh_b200 import _lib, build

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(REPO, "include")


def test_device_header_compiles_alone():
    nvcc = build.nvcc_path()
    if nvcc is None:
        pytest.skip("nvcc not present")
    src = ('#include "tinybvh_b200_device.cuh"\n'
           "__global__ void k( const tbvh_view v, tbvh::Ray* r, unsigned* bits )\n"
           "{\n"
           "    tbvh::Ray x = r[threadIdx.x];\n"
           "    tbvh::intersect_bvh( v, x ); tbvh::intersect_cwbvh( v, x );\n"
           "    tbvh::intersect_tlas<TBVH_LAYOUT_BVH>( v, x ); tbvh::intersect_tlas<TBVH_LAYOUT_CWBVH>( v, x );\n"
           "    r[threadIdx.x] = x;\n"
           "    bits[threadIdx.x] = tbvh::isoccluded_bvh( v, x ) | tbvh::isoccluded_cwbvh( v, x ) << 1 |\n"
           "        tbvh::isoccluded_tlas<TBVH_LAYOUT_BVH>( v, x ) << 2 | tbvh::isoccluded_tlas<TBVH_LAYOUT_CWBVH>( v, x ) << 3;\n"
           "}\n")
    with tempfile.TemporaryDirectory() as d:
        cu = os.path.join(d, "alone.cu")
        open(cu, "w").write(src)
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-I" + INCLUDE, "-c", cu, "-o", os.path.join(d, "alone.o")],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr


def test_view_mirror_matches_the_c_struct():
    fields = [f[0] for f in _lib.DeviceView._fields_]
    src = "#include <stddef.h>\n#include <stdio.h>\n#include \"tinybvh_b200.h\"\nint main( void )\n{\n"
    src += '    printf( "%zu\\n", sizeof( tbvh_view ) );\n'
    for f in fields:
        src += f'    printf( "%zu\\n", offsetof( tbvh_view, {f} ) );\n'
    src += "    return 0;\n}\n"
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "probe.c"), os.path.join(d, "probe")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + INCLUDE, c, "-o", exe])
        out = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    assert out[0] == C.sizeof(_lib.DeviceView) == 64
    assert out[1:] == [getattr(_lib.DeviceView, f).offset for f in fields]
