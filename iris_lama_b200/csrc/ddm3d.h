// ddm3d.h -- lama::DynamicDistanceMap with is3d = true (include/lama/sdm/dynamic_distance_map.h) on the device.
#pragma once

#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

#include "frontend.h"
#include "patch_window.h"

namespace lama_b200 {

// One 3-D distance map in a dense directory window of dim[0] x dim[1] x dim[2] patches (at most 65 536 entries).  A patch is 32^3
// cells of 8 bytes (ddm3_core.h), 256 KiB, from a pool of pool_slots (0: one per directory entry) zeroed at creation.
// addObstacle / removeObstacle are admitted on the host (window margin and pool, Dm3Guard) and queued; update() applies the queue in
// list order and runs the brushfire, one sequential thread (k_dm3_brushfire).  Every reader applies the queue first.
class DistMap3Dev {
public:
    // setMaxDistance(l2_max) at creation (dynamic_distance_map.cpp:149-153); ceil(l2_max / resolution) must be at most 63 cells and
    // dev.pool_slots below 2^24.  Null on failure, with err and its status in *code.
    static DistMap3Dev* create(double resolution, uint32_t patch_size, double l2_max, const double center[3], const int32_t window[3],
                               const DeviceOptions& dev, std::string& err, int* code);
    ~DistMap3Dev();
    DistMap3Dev(const DistMap3Dev&) = delete;
    DistMap3Dev& operator=(const DistMap3Dev&) = delete;

    uint32_t max_sqdist() const;
    double max_distance() const;   // maxDistance (:155-158)
    double resolution() const;
    // addObstacle (remove = false) / removeObstacle (:212-242) of n cells: LAMA_ERR_WINDOW when a cell lies less than reach + 1 cells
    // inside the window, LAMA_ERR_POOL when the patches the batch can reach could exceed the free slots; the map is then unchanged.
    int add_remove(const uint32_t* cells_xyz, int n, bool remove);
    // update() (:160-197); *processed (may be NULL) = its return value
    int update(uint32_t* processed);
    // distance(Vector3d, gradient) (:93-133) of n world points; gradient (n x 3) may be NULL
    int distance(const double* pts_xyz, int n, double* dist, double* gradient);
    // distance(Vector3ui) (:140-147) of n cells
    int cell_distance(const uint32_t* cells_xyz, int n, double* dist);
    int bounds(uint32_t mn[3], uint32_t mx[3], int* patches);
    // the box lo + [0, size), x fastest, then y, then z: cell words (ddm3_core.h layout; 0 where no patch) and known bits (either NULL)
    int export_box(const uint32_t lo[3], const int32_t size[3], uint64_t* words, uint8_t* known);
    int write(const std::string& path);
    int read(const std::string& path);
    // the z-slice image of sdm::export_to_png(dm, file, zed) (export.cpp:74-96): dims = {width, height}; pixels when cap is enough
    int export_image(double zed, uint8_t* pixels, size_t cap, int dims[2]);
    // ms / launches: [0] update (brushfire launches, queue flushes included), [1] distance, [2] cell_distance and export
    void kernel_times(double ms[3], uint64_t launches[3]) const;
    // {brushfire launches, heap growths, raise heap capacity, lower heap capacity}
    void run_stats(uint64_t out[4]) const;
    const std::string& error() const { return err_; }

    // ---- for OccMap3Dev::insert_point_clouds_dm3 (om3d.cu), which drives the map through these ----------------------------------------
    struct Coupling {
        int device;
        void* stream;          // cudaStream_t
        double resolution;
        PatchWindow win;
        int reach;             // R = ceil(l2_max * scale)
        const int32_t* dir;    // device directory and pool (ddm3_core.h cells)
        uint64_t* cells;
    };
    Coupling coupling() const;
    // the pool check of a batch whose distance-map ops may fall anywhere in the marked directory entries (Dm3Guard::admit_entries):
    // LAMA_ERR_POOL, or LAMA_OK with *next the reachable entries to commit once the batch is admitted
    int admit_entries(const std::vector<uint32_t>& marks, std::vector<uint8_t>& next);
    void commit_reachable(std::vector<uint8_t>& next);
    // applies the queued ops without update() (every reader does this first)
    int flush();
    // allocates the marked entries that have no patch, ascending directory index, and records `done` (a cudaEvent_t) on the map's
    // stream; the caller admitted them (admit_entries), so the pool holds them
    int alloc_entries(const std::vector<uint32_t>& marks, void* done);
    // After `wait` (a cudaEvent_t, may be null): the device op list ops (kDm3OpWords words per op) cut into segments ending at seg_end,
    // applied and updated segment by segment (Brushfire3::run_segments); processed[k] = update()'s count of segment k.
    int run_segments(const uint32_t* ops, const std::vector<uint32_t>& seg_end, uint32_t* processed, void* wait);

private:
    DistMap3Dev() = default;
    int run(bool do_update, uint32_t* processed);
    int drive(const uint32_t* ops, uint32_t n_ops, bool do_update, const uint32_t* seg_end, uint32_t n_seg, uint32_t* seg_processed);
    struct Impl;
    Impl* d_ = nullptr;
    std::string err_;
};

}  // namespace lama_b200
