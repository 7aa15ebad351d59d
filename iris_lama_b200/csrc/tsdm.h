// tsdm.h -- lama::TruncatedSignedDistanceMap (include/lama/sdm/truncated_signed_distance_map.h) on the device.
#pragma once

#include <cstddef>
#include <cstdint>
#include <string>

#include "frontend.h"

namespace lama_b200 {

// One map in a dense directory window of dim[0] x dim[1] x dim[2] patches (dim[2] = 1 in 2-D).  A patch is 32 x 32 (x 32 in 3-D)
// cells of {float distance; float weight} plus one "on" bit per cell (the Container bitmask).  Patches come from a pool of
// pool_slots (0: one per directory entry, so a full window cannot run out).
class TsdmDev {
public:
    static TsdmDev* create(double resolution, uint32_t patch_size, bool is3d, const double center[3], const int32_t window[3],
                           const DeviceOptions& dev, std::string& err);
    ~TsdmDev();
    TsdmDev(const TsdmDev&) = delete;
    TsdmDev& operator=(const TsdmDev&) = delete;

    // n_clouds calls of insertPointCloud in order; inserted[k] (may be NULL) = its return value.  A hit or walked cell outside the
    // window fails with LAMA_ERR_WINDOW (and a full pool with LAMA_ERR_POOL) before anything is written.
    int insert_point_clouds(const double* pts, const int64_t* offsets, int n_clouds, const double* origins, const double* quats, uint64_t* inserted);
    int distance(const double* pts, int n, double* dist, double* grad);
    int bounds(uint32_t mn[3], uint32_t mx[3], int* patches) const;
    int export_box(const uint32_t lo[3], const int32_t size[3], float* dist, float* weight, uint8_t* on);
    // toMesh: 3 unshared vertices per triangle (index[i] = i); vertices == NULL or cap too small: only *n_vertices
    int to_mesh(float* vertices, size_t cap, size_t* n_vertices);
    void set_max_distance(double d);
    double max_distance() const;
    double resolution() const;
    // ms / launches: [0] insert_point_clouds, [1] distance, [2] to_mesh (times only with dev.timing)
    void kernel_times(double ms[3], uint64_t launches[3]) const;
    const std::string& error() const { return err_; }

private:
    TsdmDev() = default;
    struct Impl;
    Impl* d_ = nullptr;
    std::string err_;
};

}  // namespace lama_b200
