"""CPU oracle of the reference's 3-D occupancy maps (FrequencyOccupancyMap / ProbabilisticOccupancyMap with is3d = true, the insertion
loop of GraphSlam2D::generateOccupancyMap, Map::write, the z-slice image of sdm::export_to_png), plus a host build of the device core
(iris_lama_b200/csrc/om3d_core.h) for bit-for-bit comparison.

TEST INFRASTRUCTURE ONLY.  tests/emu/occ3d_oracle.cpp and tests/emu/occ3d_emu.cpp are compiled on first use into a temporary directory.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OFFSET = 1321122 * 32
KINDS = {"frequency": 0, "logodds": 1}
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="occ3d_oracle_"), "libocc3d_oracle.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-Wall", "-shared", "-o", so,
                               os.path.join(HERE, "emu", "occ3d_oracle.cpp"), os.path.join(HERE, "emu", "occ3d_emu.cpp")])
        L = C.CDLL(so)
        for f in ("o3o_create", "o3e_create"):
            getattr(L, f).restype = C.c_void_p
            getattr(L, f).argtypes = [C.c_double, C.c_int]
        for f in ("o3o_insert", "o3e_insert"):
            getattr(L, f).restype = C.c_uint64
        L.o3o_image.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _vp(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def clouds_arrays(clouds):
    clouds = [np.ascontiguousarray(c, np.float64).reshape(-1, 3) for c in clouds]
    off = np.zeros(len(clouds) + 1, np.int64)
    off[1:] = np.cumsum([len(c) for c in clouds])
    return np.ascontiguousarray(np.concatenate(clouds) if clouds else np.zeros((0, 3))), off


def w2m(resolution, pts):
    """Map::w2m on all three axes (the oracle's arithmetic: p * scale + offset, + 0.5, truncated)"""
    p = np.asarray(pts, np.float64).reshape(-1, 3)
    return ((p * (1.0 / resolution) + float(OFFSET)) + 0.5).astype(np.uint32)


class _Base:
    prefix = None

    def __init__(self, resolution, kind="frequency"):
        self.resolution = resolution
        self.kind = kind
        self.h = C.c_void_p(getattr(lib(), self.prefix + "create")(resolution, KINDS[kind]))

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            getattr(_lib, self.prefix + "destroy")(self.h)
            self.h = None

    def _fn(self, name):
        return getattr(lib(), self.prefix + name)

    def insertPointClouds(self, clouds, origins=None, quats=None, full=True):
        p, off = clouds_arrays(clouds)
        o = None if origins is None else np.ascontiguousarray(origins, np.float64).reshape(-1, 3)
        q = None if quats is None else np.ascontiguousarray(quats, np.float64).reshape(-1, 4)
        return int(self._fn("insert")(self.h, _vp(p), _vp(off), C.c_int(len(off) - 1), _vp(o), _vp(q), C.c_int(1 if full else 0)))

    def apply(self, cells, ops):
        c = np.ascontiguousarray(cells, np.uint32).reshape(-1, 3)
        o = np.ascontiguousarray(np.broadcast_to(np.asarray(ops, np.uint8), (len(c),)))
        changed = np.zeros(len(c), np.uint8)
        self._fn("apply")(self.h, _vp(c), _vp(o), C.c_int(len(c)), _vp(changed))
        return changed.astype(bool)

    def setFree(self, cells):
        return self.apply(cells, 0)

    def setOccupied(self, cells):
        return self.apply(cells, 1)

    def setUnknown(self, cells):
        return self.apply(cells, 2)

    def query(self, cells):
        c = np.ascontiguousarray(cells, np.uint32).reshape(-1, 3)
        prob, flags = np.zeros(len(c)), np.zeros(len(c), np.uint8)
        self._fn("query")(self.h, _vp(c), C.c_int(len(c)), _vp(prob), _vp(flags))
        return prob, flags

    def prune(self):
        self._fn("prune")(self.h)

    def export(self, lo, size):
        lo = np.ascontiguousarray(lo, np.uint32)
        sz = np.ascontiguousarray(size, np.int32)
        shape = (int(sz[2]), int(sz[1]), int(sz[0]))
        w, k = np.zeros(shape, np.uint32), np.zeros(shape, np.uint8)
        self._fn("export")(self.h, _vp(lo), _vp(sz), _vp(w), _vp(k))
        return dict(word=w, known=k)


class Oracle(_Base):
    """the reference classes restated on the CPU"""
    prefix = "o3o_"

    def bounds(self):
        mn, mx = np.zeros(3, np.uint32), np.zeros(3, np.uint32)
        n = lib().o3o_bounds(self.h, _vp(mn), _vp(mx))
        return n, mn, mx

    def write(self, path):
        return lib().o3o_write(self.h, str(path).encode()) == 1

    def exportImage(self, zed=0.0):
        dims = np.zeros(2, np.int32)
        lib().o3o_image(self.h, C.c_double(zed), None, _vp(dims))
        out = np.zeros((int(dims[1]), int(dims[0])), np.uint8)
        if out.size:
            lib().o3o_image(self.h, C.c_double(zed), _vp(out), _vp(dims))
        return out


class Emu(_Base):
    """om3d_core.h run sequentially on the host"""
    prefix = "o3e_"
