// om3d.h -- lama::FrequencyOccupancyMap / lama::ProbabilisticOccupancyMap with is3d = true (include/lama/sdm/*_occupancy_map.h) on
// the device.
#pragma once

#include <cstddef>
#include <cstdint>
#include <string>

#include "frontend.h"

namespace lama_b200 {

// One 3-D occupancy map in a dense directory window of dim[0] x dim[1] x dim[2] patches (at most 65 536 entries).  A patch is
// 32 x 32 x 32 cells of 4 bytes ({uint16 occupied; uint16 visited} or a float log-odds) plus one known bit per cell (the Container
// mask), 132 KiB in all.  Patches come from a pool of pool_slots (0: one per directory entry).
class OccMap3Dev {
public:
    // kind: kOm3Frequency or kOm3LogOdds (om3d_core.h)
    static OccMap3Dev* create(double resolution, uint32_t patch_size, int kind, const double center[3], const int32_t window[3],
                              const DeviceOptions& dev, std::string& err);
    ~OccMap3Dev();
    OccMap3Dev(const OccMap3Dev&) = delete;
    OccMap3Dev& operator=(const OccMap3Dev&) = delete;

    // generateOccupancyMap's loop body for every point of n_clouds clouds in order; *cells (may be NULL) = the cell updates made.
    // A cell outside the window fails with LAMA_ERR_WINDOW, a full pool with LAMA_ERR_POOL, before anything is written.
    int insert_point_clouds(const double* pts, const int64_t* offsets, int n_clouds, const double* origins, const double* quats, bool full,
                            uint64_t* cells);
    // setFree / setOccupied / setUnknown (kOm3Set*) of n cells in list order; changed[i] (may be NULL) = the return value of op i
    int apply(const uint32_t* cells_xyz, const uint8_t* ops, int n, uint8_t* changed);
    // getProbability and the isFree / isOccupied / isUnknown flags (bits 0 / 1 / 2) of n cells
    int query(const uint32_t* cells_xyz, int n, double* prob, uint8_t* flags);
    int prune();
    int bounds(uint32_t mn[3], uint32_t mx[3], int* patches) const;
    // the box lo + [0, size), x fastest, then y, then z: cell words and known bits (either may be NULL)
    int export_box(const uint32_t lo[3], const int32_t size[3], uint32_t* words, uint8_t* known);
    int write(const std::string& path);
    int read(const std::string& path);
    // the z-slice image of sdm::export_to_png (export.cpp:46-72): dims = {width, height}; pixels written when cap is large enough
    int export_image(double zed, uint8_t* pixels, size_t cap, int dims[2]);
    int kind() const;
    double resolution() const;
    // ms / launches: [0] insert_point_clouds, [1] apply, [2] query (times only with dev.timing)
    void kernel_times(double ms[3], uint64_t launches[3]) const;
    const std::string& error() const { return err_; }

private:
    OccMap3Dev() = default;
    struct Impl;
    Impl* d_ = nullptr;
    std::string err_;
};

}  // namespace lama_b200
