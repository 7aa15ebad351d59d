// patch_window.h -- the dense directory window of the device patch stores (TsdmDev, OccMap3Dev, DistMap3Dev): a directory index per
// patch and a cell index per cell.  Plain C++ usable from host and device.
#pragma once

#include "lama_core.h"

namespace lama_b200 {

// dim[0] x dim[1] x dim[2] patches from patch coordinates base (cell >> 5); dim[2] == 1 and z ignored in 2-D (MASK3D, map.h:182-189)
struct PatchWindow {
    int32_t base[3];
    int32_t dim[3];
    int is3d;
};
// directory index (x fastest, then y, then z), or -1 outside the window
LAMA_HD int window_dir_index(const PatchWindow& w, uint32_t x, uint32_t y, uint32_t z)
{
    const int px = (int)(x >> kPatchLog2) - w.base[0], py = (int)(y >> kPatchLog2) - w.base[1];
    const int pz = w.is3d ? (int)(z >> kPatchLog2) - w.base[2] : 0;
    if ((unsigned)px >= (unsigned)w.dim[0] || (unsigned)py >= (unsigned)w.dim[1] || (unsigned)pz >= (unsigned)w.dim[2]) return -1;
    return (pz * w.dim[1] + py) * w.dim[0] + px;
}
// Map::m2c (map.h:182-189)
LAMA_HD uint32_t window_cell_index(uint32_t x, uint32_t y, uint32_t z, int is3d)
{
    const uint32_t m = kPatchLen - 1;
    return (x & m) | ((y & m) << kPatchLog2) | (is3d ? (z & m) << (2 * kPatchLog2) : 0u);
}
// directory index -> the anchor cell of its patch (z = 0 in 2-D, where base[2] = 0 and dim[2] = 1)
LAMA_HD void window_anchor(const PatchWindow& w, int i, uint32_t a[3])
{
    const int p[3] = {i % w.dim[0], (i / w.dim[0]) % w.dim[1], i / (w.dim[0] * w.dim[1])};
    for (int k = 0; k < 3; ++k) a[k] = (uint32_t)(w.base[k] + p[k]) << kPatchLog2;
}

}  // namespace lama_b200
