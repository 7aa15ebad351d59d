"""CPU test of the sector-aligned segment partition k_raycast uses for the beams of x-major beam groups: a host build of ray_core.h
(tests/emu/seg_align_emu.cpp) against Map::computeRay's iterative walk (map.cpp:198-227)."""
import ctypes as C
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("seg_align_emu") / "libseg_align_emu.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-shared", "-o", so,
                           os.path.join(HERE, "emu", "seg_align_emu.cpp")])
    L = C.CDLL(so)
    L.emu_seg_align_check.restype = C.c_int
    L.emu_seg_align_check.argtypes = [C.c_int, C.c_uint32, C.c_uint32, C.c_int, C.c_int]
    return L


# the centre's x mod 8 sets the shift of every beam from it: eight centres give every shift 0 .. 7 in both x directions
@pytest.mark.parametrize("centre", range(2000, 2008))
def test_aligned_segments_cover_every_step_once_in_sector_octets(emu, centre):
    """Every step exactly once on the reference's cell, each strided instruction of an x-major beam inside one aligned octet of x, and
    the look-ahead inside the bounding box of the beam's end cells: all beams from one centre into a 401^2 box (odd and even lengths,
    n = 0, 1, diagonals)"""
    assert emu.emu_seg_align_check(200, centre, 0, 0, 0) == 0


def test_aligned_segments_random_beams(emu):
    assert emu.emu_seg_align_check(0, 0, 5, 50000, 2048) == 0   # dir_dim 64 windows
    assert emu.emu_seg_align_check(0, 0, 6, 50000, 4096) == 0   # the largest window (dir_dim 128)
