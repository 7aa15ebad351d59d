"""CPU oracle of lama::TruncatedSignedDistanceMap (src/sdm/truncated_signed_distance_map.cpp), toMesh and sdm::export_to_ply, plus a
host build of the device fusion core (iris_lama_b200/csrc/tsdm_core.h) for bit-for-bit comparison.

TEST INFRASTRUCTURE ONLY.  tests/emu/tsdm_oracle.cpp and tests/emu/tsdm_emu.cpp are compiled on first use into a temporary directory.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OFFSET = 1321122 * 32
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="tsdm_oracle_"), "libtsdm_oracle.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-Wall", "-shared", "-o", so,
                               os.path.join(HERE, "emu", "tsdm_oracle.cpp"), os.path.join(HERE, "emu", "tsdm_emu.cpp")])
        L = C.CDLL(so)
        for f in ("tso_create", "tse_create"):
            getattr(L, f).restype = C.c_void_p
            getattr(L, f).argtypes = [C.c_double, C.c_int]
        L.tso_mesh.restype = C.c_size_t
        _lib = L
    return _lib


def _vp(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def clouds_arrays(clouds):
    clouds = [np.ascontiguousarray(c, np.float64).reshape(-1, 3) for c in clouds]
    off = np.zeros(len(clouds) + 1, np.int64)
    off[1:] = np.cumsum([len(c) for c in clouds])
    return np.ascontiguousarray(np.concatenate(clouds) if clouds else np.zeros((0, 3))), off


class _Base:
    prefix = None

    def __init__(self, resolution, is3d=False):
        self.resolution = resolution
        self.is3d = is3d
        self.h = C.c_void_p(getattr(lib(), self.prefix + "create")(resolution, 1 if is3d else 0))

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            getattr(_lib, self.prefix + "destroy")(self.h)
            self.h = None

    def _fn(self, name):
        return getattr(lib(), self.prefix + name)

    def insertPointClouds(self, clouds, origins=None, quats=None):
        p, off = clouds_arrays(clouds)
        o = None if origins is None else np.ascontiguousarray(origins, np.float64).reshape(-1, 3)
        q = None if quats is None else np.ascontiguousarray(quats, np.float64).reshape(-1, 4)
        out = np.zeros(len(off) - 1, np.uint64)
        self._fn("insert")(self.h, _vp(p), _vp(off), C.c_int(len(off) - 1), _vp(o), _vp(q), _vp(out))
        return out

    def insertPointCloud(self, points, origin=None, quat=None):
        return int(self.insertPointClouds([points], None if origin is None else [origin], None if quat is None else [quat])[0])

    def export(self, lo, size):
        lo = np.ascontiguousarray(lo, np.uint32)
        sz = np.ascontiguousarray(size, np.int32)
        shape = (int(sz[2]), int(sz[1]), int(sz[0]))
        o = dict(distance=np.zeros(shape, np.float32), weight=np.zeros(shape, np.float32), on=np.zeros(shape, np.uint8))
        self._fn("export")(self.h, _vp(lo), _vp(sz), _vp(o["distance"]), _vp(o["weight"]), _vp(o["on"]))
        return o

    def distance(self, points, gradient=False):
        p = np.ascontiguousarray(points, np.float64).reshape(-1, 3)
        n = len(p)
        dist, grad = np.zeros(n), np.zeros((n, 3))
        self._fn("distance")(self.h, _vp(p), C.c_int(n), _vp(dist), _vp(grad))
        return (dist, grad) if gradient else dist


class Oracle(_Base):
    """the reference class restated on the CPU"""
    prefix = "tso_"

    def setMaxDistance(self, d):
        lib().tso_set_max_distance(self.h, C.c_double(d))

    def integrate(self, origin, hit):
        o, h = np.ascontiguousarray(origin, np.float64), np.ascontiguousarray(hit, np.float64)
        lib().tso_integrate(self.h, _vp(o), _vp(h))

    def bounds(self):
        mn, mx = np.zeros(3, np.uint32), np.zeros(3, np.uint32)
        n = lib().tso_bounds(self.h, _vp(mn), _vp(mx))
        return n, mn, mx

    def toMesh(self):
        n = lib().tso_mesh(self.h, None, C.c_size_t(0))
        v = np.zeros((n, 3), np.float32)
        if n:
            lib().tso_mesh(self.h, _vp(v), C.c_size_t(n))
        return v

    def write_ply(self, path):
        return lib().tso_write_ply(self.h, str(path).encode()) == 1


class Emu(_Base):
    """tsdm_core.h run sequentially on the host"""
    prefix = "tse_"

    def cube(self, cell, table):
        out = np.zeros((16, 3), np.float32)
        cfg = lib().tse_cube(self.h, C.c_uint32(int(cell[0])), C.c_uint32(int(cell[1])), C.c_uint32(int(cell[2])), _vp(table), _vp(out))
        return cfg, out


def mc_table():
    """the product's generated triangle table: (tri (256, row) int8, -1 terminated; ntri (256,))"""
    row = lib().tso_mc_row()
    tri, ntri = np.zeros((256, row), np.int8), np.zeros(256, np.uint8)
    lib().tso_mc_table(_vp(tri), _vp(ntri))
    return tri, ntri
