"""CPU test of ray_core.h StrideWalk, the walk k_raycast uses for the segments of x-major beam groups after the first: a host
build of the same header (tests/emu/stride_walk_emu.cpp) against Map::computeRay's iterative walk (map.cpp:198-227)."""
import ctypes as C
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("stride_walk_emu") / "libstride_walk_emu.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-shared", "-o", so,
                           os.path.join(HERE, "emu", "stride_walk_emu.cpp")])
    L = C.CDLL(so)
    L.emu_stridewalk_check.restype = C.c_int
    L.emu_stridewalk_check.argtypes = [C.c_int, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_int]
    return L


# stride 1 is the walk of y-major groups, 8 the one k_raycast uses for x-major groups; 2, 3 and 4 cover strides that do not divide
# the segment length evenly and strides shorter than the kernel's
@pytest.mark.parametrize("stride", [1, 2, 3, 4, 8])
def test_stride_walk_visits_the_iterative_bresenham_cells(emu, stride):
    """For every segment and start offset: exactly the cells of the reference walk at the steps congruent to the offset, and the
    look-ahead step of the kernel's loop never leaves the bounding box of the beam's end cells"""
    assert emu.emu_stridewalk_check(150, 0, 0, 0, 64, stride) == 0      # all 301^2 beams from one centre incl. n = 0, 1, diagonals
    assert emu.emu_stridewalk_check(40, 0, 0, 0, 7, stride) == 0        # odd segment length
    assert emu.emu_stridewalk_check(0, 3, 20000, 2048, 64, stride) == 0  # random beams in dir_dim 64 windows
    assert emu.emu_stridewalk_check(0, 4, 20000, 4096, 64, stride) == 0  # the largest window (dir_dim 128)
