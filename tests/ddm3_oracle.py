"""CPU oracle of the reference's 3-D DynamicDistanceMap (DynamicDistanceMap with is3d = true: the six-neighbour brushfire, distance
queries, Map::write, the z-slice image of sdm::export_to_png), plus a host build of the device core (iris_lama_b200/csrc/ddm3_core.h)
for bit-for-bit comparison, and the sanitizer build of the standalone comparison (tests/emu/ddm3_check.cpp).

TEST INFRASTRUCTURE ONLY.  tests/emu/ddm3_oracle.cpp and tests/emu/ddm3_emu.cpp are compiled on first use into a temporary directory.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
OFFSET = 1321122 * 32
UC = 2642244
_lib = None
_check = {}


def _cxx():
    return os.environ.get("CXX", "g++")


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="ddm3_oracle_"), "libddm3_oracle.so")
        subprocess.check_call([_cxx(), "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-Wall", "-shared", "-o", so,
                               os.path.join(EMU, "ddm3_oracle.cpp"), os.path.join(EMU, "ddm3_emu.cpp")])
        L = C.CDLL(so)
        L.d3o_create.restype = C.c_void_p
        L.d3o_create.argtypes = [C.c_double, C.c_double]
        L.d3e_create.restype = C.c_void_p
        L.d3e_create.argtypes = [C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_int]
        L.d3o_max_distance.restype = C.c_double
        L.d3e_error.restype = C.c_char_p
        for f in ("d3o_update", "d3o_max_sqdist"):
            getattr(L, f).restype = C.c_uint32
        _lib = L
    return _lib


def check_binary(sanitize=True):
    """the standalone emu-vs-oracle comparison, built with -fsanitize=address,undefined when `sanitize`"""
    if sanitize not in _check:
        exe = os.path.join(tempfile.mkdtemp(prefix="ddm3_check_"), "ddm3_check")
        flags = ["-O1", "-g", "-fno-omit-frame-pointer", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"] if sanitize else ["-O2"]
        srcs = [os.path.join(EMU, f) for f in ("ddm3_check.cpp", "ddm3_oracle.cpp", "ddm3_emu.cpp")]
        # not every compiler install ships the sanitizer runtimes: the first one that links the build is taken
        compilers = [_cxx(), "g++", "/usr/bin/g++", "clang++"] if sanitize else [_cxx()]
        errors = []
        for cxx in dict.fromkeys(compilers):
            r = subprocess.run([cxx, "-std=c++17", "-ffp-contract=off", "-Wall", *flags, "-o", exe, *srcs], capture_output=True, text=True)
            if r.returncode == 0:
                break
            errors.append(f"{cxx}: {r.stderr[-400:]}")
        else:
            raise RuntimeError("no compiler could build ddm3_check:\n" + "\n".join(errors))
        _check[sanitize] = exe
    return _check[sanitize]


def _vp(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def ops_array(cells, kind):
    """(n, 4) uint32 ops: x, y, z, kind (0 addObstacle, 1 removeObstacle)"""
    c = np.ascontiguousarray(cells, np.uint32).reshape(-1, 3)
    return np.ascontiguousarray(np.c_[c, np.full(len(c), kind, np.uint32)])


def scenario_bytes(steps):
    """steps: ("add" | "remove", cells) or ("update",) -> the scenario file of ddm3_check.cpp"""
    words = []
    for s in steps:
        if s[0] == "update":
            words.append(np.array([1], np.uint32))
        else:
            o = ops_array(s[1], 1 if s[0] == "remove" else 0)
            words += [np.array([0, len(o)], np.uint32), o.ravel()]
    return np.concatenate(words).astype("<u4").tobytes() if words else b""


class _Base:
    prefix = None

    def _fn(self, name):
        return getattr(lib(), self.prefix + name)

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            getattr(_lib, self.prefix + "destroy")(self.h)
            self.h = None

    def addObstacle(self, cells):
        return self.apply(ops_array(cells, 0))

    def removeObstacle(self, cells):
        return self.apply(ops_array(cells, 1))

    def distance(self, pts):
        p = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
        d, g = np.zeros(len(p)), np.zeros((len(p), 3))
        self._fn("distance")(self.h, _vp(p), C.c_int(len(p)), _vp(d), _vp(g))
        return d, g

    def cellDistance(self, cells):
        c = np.ascontiguousarray(cells, np.uint32).reshape(-1, 3)
        d = np.zeros(len(c))
        self._fn("cell_distance")(self.h, _vp(c), C.c_int(len(c)), _vp(d))
        return d

    def bounds(self):
        mn, mx = np.zeros(3, np.uint32), np.zeros(3, np.uint32)
        n = self._fn("bounds")(self.h, _vp(mn), _vp(mx))
        return n, mn, mx

    def patch_ids(self):
        n = self.bounds()[0]
        ids = np.zeros(max(n, 1), np.uint64)
        self._fn("patch_ids")(self.h, _vp(ids))
        return sorted(int(i) for i in ids[:n])

    def export(self, lo, size):
        lo = np.ascontiguousarray(lo, np.uint32)
        sz = np.ascontiguousarray(size, np.int32)
        shape = (int(sz[2]), int(sz[1]), int(sz[0]))
        w, k = np.zeros(shape, np.uint64), np.zeros(shape, np.uint8)
        self._fn("export")(self.h, _vp(lo), _vp(sz), _vp(w), _vp(k))
        return dict(word=w, known=k)


class Oracle(_Base):
    """the reference class restated on the CPU"""
    prefix = "d3o_"

    def __init__(self, resolution, l2_max):
        self.resolution = resolution
        self.h = C.c_void_p(lib().d3o_create(resolution, l2_max))

    @property
    def max_sqdist(self):
        return int(lib().d3o_max_sqdist(self.h))

    def maxDistance(self):
        return float(lib().d3o_max_distance(self.h))

    def apply(self, ops):
        o = np.ascontiguousarray(ops, np.uint32)
        lib().d3o_apply(self.h, _vp(o), C.c_int(len(o)))
        return 0

    def update(self):
        return int(lib().d3o_update(self.h))

    def write(self, path):
        return lib().d3o_write(self.h, str(path).encode()) == 1

    def exportImage(self, zed=0.0):
        dims = np.zeros(2, np.int32)
        lib().d3o_image(self.h, C.c_double(zed), None, _vp(dims))
        out = np.zeros((int(dims[1]), int(dims[0])), np.uint8)
        if out.size:
            lib().d3o_image(self.h, C.c_double(zed), _vp(out), _vp(dims))
        return out


class Emu(_Base):
    """ddm3_core.h run on the host, admitted and resumed as the device map does it"""
    prefix = "d3e_"

    def __init__(self, resolution, l2_max, window=(8, 8, 4), center=None, pool_slots=0):
        self.resolution = resolution
        w = np.ascontiguousarray(window, np.int32)
        c = None if center is None else np.ascontiguousarray(center, np.float64)
        self.h = C.c_void_p(lib().d3e_create(resolution, l2_max, _vp(c), _vp(w), C.c_int(pool_slots)))

    def apply(self, ops):
        """the admission, then queued: 0, -4 (window) or -5 (pool)"""
        o = np.ascontiguousarray(ops, np.uint32)
        return int(lib().d3e_apply(self.h, _vp(o), C.c_int(len(o))))

    def error(self):
        return lib().d3e_error(self.h).decode()

    def update(self):
        n = C.c_uint32(0)
        rc = lib().d3e_update(self.h, C.byref(n))
        assert rc == 0, self.error()
        return n.value

    def stats(self):
        s = np.zeros(4, np.uint64)
        lib().d3e_stats(self.h, _vp(s))
        return dict(zip(("launches", "grows", "raise_cap", "lower_cap"), s.tolist()))


def patch_anchor(pid):
    return np.array([(pid // (UC * UC)) << 5, ((pid % (UC * UC)) // UC) << 5, (pid % UC) << 5], np.uint32)


def same_maps(a, b, patch_ids=None):
    """a (an Oracle or Emu) and b: `patch_ids(b)` lists b's patches when b has no patch_ids().  Every cell (the 64-bit word: offsets, flags with the known bit, sqdist) of every patch, the patch set and the bounds"""
    ia = a.patch_ids()
    ib = patch_ids(b) if patch_ids else b.patch_ids()
    assert ia == ib, (len(ia), len(ib))
    na, mna, mxa = a.bounds()
    nb, mnb, mxb = b.bounds()
    assert na == nb and (na == 0 or (np.array_equal(mna, mnb) and np.array_equal(mxa, mxb)))
    for pid in ia:
        lo = patch_anchor(pid)
        ea, eb = a.export(lo, (32, 32, 32)), b.export(lo, (32, 32, 32))
        assert np.array_equal(ea["known"], eb["known"]), pid
        assert np.array_equal(ea["word"], eb["word"]), pid


def read_sdm(path):
    """(header bytes, params, {patch id: (cells bytes, mask bytes)}) of a 3-D distance .sdm file"""
    data = open(path, "rb").read()
    n = int(np.frombuffer(data[16:24], np.uint64)[0])
    params = data[32:36]
    patch = 8 + 32768 * 10 + 512 * 8
    out = {}
    for i in range(n):
        o = 36 + i * patch
        pid = int(np.frombuffer(data[o:o + 8], np.uint64)[0])
        out[pid] = (data[o + 8:o + 8 + 327680], data[o + 8 + 327680:o + patch])
    assert len(data) == 36 + n * patch
    return data[:32], params, out
