"""CPU oracle of GraphSlam2D's global maps: generateOccupancyMap (src/graph_slam2d.cpp:131-164), FrequencyOccupancyMap::prune
(src/sdm/frequency_occupancy_map.cpp:149-158) and generateCoarseDistanceMap (:166-186).

TEST INFRASTRUCTURE ONLY.  The map code is tests/emu/global_map_oracle.cpp on the oracle's FrequencyOccupancyMap, compiled on first
use into a temporary directory; the graph bookkeeping extends oracle/graph_slam_oracle.py with mapping_keyid.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import graph_slam_oracle as gso
from oracle import pyoracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
OFFSET = 1321122 * 32
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="global_map_oracle_"), "libglobal_map_oracle.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-Wall", "-shared",
                               "-o", so, os.path.join(HERE, "emu", "global_map_oracle.cpp")])
        L = C.CDLL(so)
        L.gmo_create.restype = C.c_void_p
        L.gmo_create.argtypes = [C.c_double, C.c_uint32]
        L.gmo_insert_scans.restype = C.c_uint64
        for f in ("gmo_destroy", "gmo_prune", "gmo_bounds", "gmo_patches", "gmo_export", "gmo_query", "gmo_write", "gmo_image", "gmo_insert_scans"):
            getattr(L, f).argtypes = None
        _lib = L
    return _lib


def _vp(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class OccupancyMap:
    """the oracle's FrequencyOccupancyMap with the render loop and prune"""

    def __init__(self, resolution, patch=32):
        self.resolution = resolution
        self.h = C.c_void_p(lib().gmo_create(resolution, patch))

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.gmo_destroy(self.h)
            self.h = None

    def insert_scans(self, scans, states, full, origins=None, quats=None, thetas=None):
        """states (S, 4) SE2 {cos, sin, x, y}; thetas (S,) replaces atan2(sin, cos) when given (poses read back as x, y, theta)"""
        scans = [np.ascontiguousarray(s, np.float64).reshape(-1, 3) for s in scans]
        off = np.zeros(len(scans) + 1, np.int64)
        off[1:] = np.cumsum([len(s) for s in scans])
        pts = np.ascontiguousarray(np.concatenate(scans) if scans else np.zeros((0, 3)))
        st = np.ascontiguousarray(states, np.float64).reshape(-1, 4)
        o = None if origins is None else np.ascontiguousarray(origins, np.float64).reshape(-1, 3)
        q = None if quats is None else np.ascontiguousarray(quats, np.float64).reshape(-1, 4)
        th = None if thetas is None else np.ascontiguousarray(thetas, np.float64)
        return int(lib().gmo_insert_scans(self.h, _vp(pts), _vp(off), C.c_int(len(scans)), _vp(o), _vp(q), _vp(st), _vp(th), C.c_int(1 if full else 0)))

    def prune(self):
        lib().gmo_prune(self.h)

    def bounds(self):
        mn, mx = np.zeros(2, np.uint32), np.zeros(2, np.uint32)
        n = lib().gmo_bounds(self.h, _vp(mn), _vp(mx))
        return n, mn, mx

    def patches(self):
        n = lib().gmo_patches(self.h, None, C.c_int(0))
        keys = np.zeros(n, np.uint64)
        lib().gmo_patches(self.h, _vp(keys), C.c_int(n))
        return set(int(k) for k in keys)

    def export(self, x0, y0, w, h):
        out = dict(occupied=np.zeros((h, w), np.uint16), visited=np.zeros((h, w), np.uint16), known=np.zeros((h, w), np.uint8))
        lib().gmo_export(self.h, C.c_uint32(x0), C.c_uint32(y0), C.c_int(w), C.c_int(h), _vp(out["occupied"]), _vp(out["visited"]), _vp(out["known"]))
        return out

    def query(self, cells):
        c = np.ascontiguousarray(cells, np.uint32)
        n = c.size // 2
        prob, flags = np.zeros(n), np.zeros(n, np.uint8)
        lib().gmo_query(self.h, _vp(c), C.c_int(n), _vp(prob), _vp(flags))
        return prob, flags

    def write(self, path):
        return lib().gmo_write(self.h, str(path).encode()) == 1

    def image(self):
        dims = (C.c_int * 2)()
        lib().gmo_image(self.h, None, C.c_size_t(0), dims)
        out = np.zeros((dims[1], dims[0]), np.uint8)
        if out.size:
            lib().gmo_image(self.h, _vp(out), C.c_size_t(out.size), dims)
        return out


def patch_keys(mn, mx, present):
    """Map::m2p keys (map.h:153-161) of the patches flagged in a dense present[(h, w)] window starting at cell mn"""
    keys = set()
    for py in range(0, present.shape[0], 32):
        for px in range(0, present.shape[1], 32):
            if present[py:py + 32, px:px + 32].any():
                keys.add(((int(mn[0]) + px) >> 5) * 2642244 + ((int(mn[1]) + py) >> 5))
    return keys


def coarse_obstacles(occ, dm_known, mn, fine_res, coarse_res=0.1):
    """generateCoarseDistanceMap's obstacle list (:171-181): occ / dm_known planes of the inner Slam2D over a patch-aligned window
    starting at cell mn; cells visited in ascending directory index (patch rows bottom up, patches left to right), then container
    order (x fastest) -- the reference's unordered_map order cannot be reproduced, so this order is the defined one"""
    h, w = dm_known.shape
    out = []
    fine_scale, coarse_scale = 1.0 / fine_res, 1.0 / coarse_res
    for py in range(0, h, 32):
        for px in range(0, w, 32):
            for y in range(py, py + 32):
                for x in range(px, px + 32):
                    if not dm_known[y, x]:
                        continue
                    o, v = int(occ["occupied"][y, x]), int(occ["visited"][y, x])
                    if not (occ["known"][y, x] and v != 0 and o / v > 0.25):     # isOccupied (frequency_occupancy_map.cpp:128-134)
                        continue
                    cell = []
                    for c in (int(mn[0]) + x, int(mn[1]) + y):
                        wpos = (float(c) - OFFSET) / fine_scale                  # m2w (map.h:147-148)
                        cell.append(int(np.uint32(wpos * coarse_scale + OFFSET + 0.5)))   # w2m (map.h:125-126)
                    out.append(cell)
    return np.array(out, np.uint32).reshape(-1, 2)


class GraphSlam2D(gso.GraphSlam2D):
    """graph_slam_oracle.GraphSlam2D with mapping_keyid (reset by optimizePoseGraph, :428) and the two generators"""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.resolution = kw.get("resolution", 0.05)
        self.mapping_keyid = 0
        self.occ = None

    def optimizePoseGraph(self):
        out = super().optimizePoseGraph()
        if out is not None:
            self.mapping_keyid = 0
        return out

    def generateOccupancyMap(self, full=False):
        if self.mapping_keyid == 0:
            self.occ = OccupancyMap(self.resolution if full else 0.1)
        keys = self.keys[self.mapping_keyid:]
        self.occ.insert_scans([k["pts"] for k in keys], [k["pose"] for k in keys], full)
        self.occ.prune()
        self.mapping_keyid = len(self.keys)
        return self.occ

    def generateCoarseDistanceMap(self):
        """-> (oracle DDM, update() return value)"""
        n1, a0, a1 = self.slam.dm_bounds()
        n0, b0, b1 = self.slam.occ_bounds()
        dm = po.DDM(0.1, 32, 5.0)
        if n0 + n1 > 0:
            mn = np.minimum(a0, b0) if n0 and n1 else (a0 if n1 else b0)
            mx = np.maximum(a1, b1) if n0 and n1 else (a1 if n1 else b1)
            w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
            known = self.slam.export_dm(mn[0], mn[1], w, h)["known"]
            occ = self.slam.export_occ(mn[0], mn[1], w, h)
            cells = coarse_obstacles(occ, known, mn, self.resolution)
            if len(cells):
                dm.add(cells)
        return dm, dm.update()
