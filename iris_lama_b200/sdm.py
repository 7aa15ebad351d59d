"""Host mirror of the reference's on-disk sparse-dense map format (".sdm"), numpy only.

Layout (src/sdm/map.cpp:490-575): IOHeader (include/lama/sdm/map.h:95-103, 32 bytes with natural padding), the concrete
map's parameters (DynamicDistanceMap: uint32 max_sqdist_, dynamic_distance_map.cpp:200-208; the occupancy maps: none), then
per patch: uint64 id = (x >> 5) * 2642244 + (y >> 5) (map.h:153-161), 1024 cells, 16 uint64 mask words (container.cpp:143-176).
3-D maps (is_3d = 1): id = ((x >> 5) * 2642244 + (y >> 5)) * 2642244 + (z >> 5), 32 768 cells, 512 mask words per patch.
The files are written by lama_*_write_map / lama_dm_write (include/lama_b200.h) and by the reference's Map::write.
"""
import numpy as np

MAGIC = 0x6D64732E
IO_VERSION = 0x0103
UNIVERSAL_CONSTANT = 2642244

HEADER = np.dtype([("magic", "<u4"), ("version", "<u2"), ("pad0", "<u2"), ("cell_size", "<u4"), ("patch_length", "<u4"), ("num_patches", "<u8"),
                   ("resolution", "<f4"), ("is_3d", "u1"), ("pad1", "u1", 3)])
assert HEADER.itemsize == 32

CELL_TYPES = {
    10: np.dtype([("ox", "<i2"), ("oy", "<i2"), ("oz", "<i2"), ("sqdist", "<u2"), ("valid", "u1"), ("queued", "u1")]),  # distance_t
    4: np.dtype([("occupied", "<u2"), ("visited", "<u2")]),                                                               # frequency (or float32 log-odds)
    1: np.dtype("i1"),                                                                                                    # SimpleOccupancyMap
}


def read_sdm(path, n_params=None):
    """-> dict(header=..., params=bytes, patches={id: (cells[volume], mask[volume // 64])}); volume = 1024, or 32 768 in a 3-D
    file; n_params defaults to 4 for 10-byte cells"""
    raw = np.fromfile(path, np.uint8)
    hdr = raw[:32].view(HEADER)[0]
    if hdr["magic"] != MAGIC or hdr["version"] != IO_VERSION:
        raise ValueError("not an sdm file of version 0x0103")
    cs = int(hdr["cell_size"])
    if n_params is None:
        n_params = 4 if cs == 10 else 0
    vol = int(hdr["patch_length"]) ** (3 if hdr["is_3d"] else 2)
    rec = 8 + vol * cs + (vol // 64) * 8
    body = raw[32 + n_params:]
    n = int(hdr["num_patches"])
    if body.size != n * rec:
        raise ValueError("patch list size %d != %d patches of %d bytes" % (body.size, n, rec))
    patches = {}
    for i in range(n):
        r = body[i * rec:(i + 1) * rec]
        pid = int(r[:8].view("<u8")[0])
        patches[pid] = (r[8:8 + vol * cs].view(CELL_TYPES[cs]).copy(), r[8 + vol * cs:].view("<u8").copy())
    return dict(header=hdr, params=raw[32:32 + n_params].tobytes(), patches=patches)


def export_to_ply(tsdm, filename):
    """sdm::export_to_ply (export.cpp:112-143): ASCII PLY of a TruncatedSignedDistanceMap's toMesh, faces written as 3 i+2 i+1 i"""
    import ctypes as C
    from . import api
    api._chk(api.lib().lama_tsdm_write_ply(tsdm.h, C.c_char_p(str(filename).encode())))
    return True


def patch_origin3(pid, patch_length=32):
    """Map::p2m (map.h:166-177) of a 3-D map: the absolute cell coordinates (x, y, z) of a patch's first cell"""
    u = UNIVERSAL_CONSTANT
    return (pid // (u * u)) * patch_length, ((pid % (u * u)) // u) * patch_length, (pid % u) * patch_length


def patch_origin(pid, patch_length=32):
    """Map::p2m (map.h:166-177): the absolute cell coordinates of a patch's first cell"""
    return (pid // UNIVERSAL_CONSTANT) * patch_length, (pid % UNIVERSAL_CONSTANT) * patch_length
