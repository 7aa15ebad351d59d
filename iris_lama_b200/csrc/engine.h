// engine.h -- host-side owner of the device-resident particle maps and the kernel pipeline.
// Plain C++ interface (no CUDA types) so the front ends and the C-ABI can be compiled by g++.
#pragma once

#include <cstdint>
#include <string>
#include <vector>

#include "lama_core.h"
#include "match_core.h"
#include "ray_core.h"

namespace lama_b200 {

struct EngineConfig {
    int device        = 0;
    int particles     = 1;      // particles resident on THIS device
    double resolution = 0.05;
    double l2_max     = 0.5;
    int dir_dim       = 64;     // directory window: dir_dim x dir_dim patches of 32 x 32 cells
    int pool_slots    = 0;      // 0 = auto (particles * 768 + 1024)
    int max_beams     = 2048;
    double center_x   = 0.0;    // world position the directory window is centred on
    double center_y   = 0.0;
    uint64_t stream   = 0;      // external cudaStream_t (0 = own non-blocking stream)
    int occupancy_kind = 0;     // 0 = FrequencyOccupancyMap (PFSlam2D, Slam2D), 1 = ProbabilisticOccupancyMap (log-odds)
    int event_cap      = 0;     // obstacle events one brushfire takes (0 = auto: max_beams rounded up to a power of two, at least 2 048)
    bool known_plane   = false; // a frequency map that keeps the Container 'known' bits in their own plane (render_scans / prune_frequency):
                                // after a prune, `known` can no longer be derived from a non-zero cell
};

struct HostMatchResult {
    SE2 state;
    double sums[kNumSums];
    uint32_t iterations, evals_ref, evals_done, pad;
};

struct HostMapStats {
    uint32_t ray_cells, log_records, events, dm_pops;
};

// The device state of an engine in a self-contained form (checkpoint.h writes and reads it).  The K slots in use are renumbered
// 0 .. K-1 in ascending order of their old slot; directory entries keep their flag bits.
struct EngineImage {
    int particles = 1, dir_dim = 64, pool_slots = 0, max_beams = 2048, occupancy_kind = 0;
    bool known_plane = false;
    double resolution = 0.05, l2_max = 0.5;
    DirWindow window{};
    uint64_t counters[3] = {0, 0, 0};      // patches allocated, detached, freed
    uint32_t used = 0;                     // K
    std::vector<int32_t> refcount;         // [K]
    std::vector<int32_t> dirs;             // [particles][n_kinds][dir_dim^2] of the current set
    // K x 4 KiB of cells, then K x 128 B of obstacle-mirror bits, then (known plane) K x 128 B of known bits
    const uint8_t* slot_bytes = nullptr;
    std::vector<uint8_t> slot_store;       // owns slot_bytes after a snapshot
    int n_kinds() const { return occupancy_kind == 1 ? 3 : 2; }
    bool has_kbits() const { return occupancy_kind == 1 || known_plane; }
    size_t slot_stride() const { return (size_t)kPatchBytes + 128 + (has_kbits() ? 128 : 0); }
};

// where the time of a snapshot / restore went (ms).  Snapshot: count, compaction, gather = CUDA events; copy = host clock of the chunked
// device -> host copy.  Restore: create = engine creation, tables = directories, reference counts, free stack and counters; copy = the
// chunked host -> device copy of the slots.
struct CheckpointTimes {
    double count_ms = 0, compact_ms = 0, gather_ms = 0, copy_ms = 0, create_ms = 0, tables_ms = 0;
};

struct KernelTimes {  // accumulated CUDA-event durations (ms) and launch counts since reset
    double match_ms = 0, raycast_ms = 0, brushfire_ms = 0, resample_ms = 0;
    uint64_t match_launches = 0, raycast_launches = 0, brushfire_launches = 0, resample_launches = 0, misc_launches = 0;
};

class Engine {
public:
    static Engine* create(const EngineConfig& cfg, std::string& err);
    ~Engine();

    const EngineConfig& config() const { return cfg_; }
    uint32_t max_sqdist() const { return max_sqdist_; }
    double logodds_threshold() const;   // ProbabilisticOccupancyMap::occ_thresh_ (probabilistic_occupancy_map.cpp:59)
    const std::string& last_error() const { return err_; }

    // Uploads one scan (N x 3 doubles, sensor origin, sensor orientation quaternion xyzw).
    int set_scan(const double* pts, int n, const double origin[3], const double quat[4], double truncated_ray, double truncated_range);
    void set_lidar_odometry_rays(bool on) { lo_ray_ = on; }   // ScanParams::lo_ray for the scans set from now on
    const ScanParams& scan_params() const;
    // Transient map (slam2d.cpp:323-379, lidar_odometry_2d.cpp:130-181): Map::deletePatchAt on the occupancy and the distance map for
    // every patch whose AABB does not meet the AABB (center, half width) -- AABB::testIntersection, include/lama/aabb.h:65-72
    int prune_outside(int particle, const double center[2], const double hwidth[2], int* removed);

    // Copies n_scans scans of n beams each into device memory once; select_staged() then makes scan `index`
    // current without any host->device transfer (inputs resident in HBM).
    int stage_scans(const double* pts, int n_scans, int n);
    int select_staged(int index, const double origin[3], const double quat[4], double truncated_ray, double truncated_range);

    // Scan matching of `count` states.  Block k uses the map of particle first_particle + k, or, with
    // shared_map, all of them use the map of first_particle.  mode 0 = solve, 1 = single evaluation.
    int match(const SE2* states, int count, int first_particle, bool shared_map, const SolverOptions& so, double meas_sigma, int mode,
              HostMatchResult* out);

    // MatchSurface2D::error() (nearest-cell RMSE of the current scan) at `count` states, maps chosen like match().
    int match_error(const SE2* states, int count, int first_particle, bool shared_map, double* out);

    // Ray-cast + distance-map update of particles [first, first+count) at the given poses.
    int update_maps(const SE2* states, int first_particle, int count, HostMapStats* out);
    // Same, but returns right after the launches; the work is collected by settle(), which every later entry point
    // calls first (errors of an asynchronous update therefore surface at the next call).
    int update_maps_async(const SE2* states, int first_particle, int count);
    int settle(HostMapStats* out, bool already_complete = false);
    // One scan of a particle filter enqueued at once: match -> ray cast -> brushfire with no host round trip in between.  The map
    // update runs on the MATCHED poses straight from the device results, i.e. BEFORE the resampling decision of this scan; a
    // resampling applied afterwards copies the updated maps, which gives the same maps as the reference's resample-then-update
    // (update(copy(m), pose) == copy(update(m, pose)), DESIGN.md 12).  Returns when the match results are on the host; the map
    // update keeps running and is collected by the next settle().  `pts` != nullptr: upload that scan first (no synchronisation).
    int step_async(const double* pts, int n, const double origin[3], const double quat[4], double truncated_ray, double truncated_range,
                   const SE2* predicted, int count, const SolverOptions& so, double meas_sigma, HostMatchResult* out);
    // The same without waiting for anything (sharded ranks): the match results stay on the device, where pack_results() turns them into
    // the exchange payload on another stream once the match has finished; collect_previous() then books the previous scan's map update.
    int step_enqueue(const double* pts, int n, const double origin[3], const double quat[4], double truncated_ray, double truncated_range,
                     const SE2* predicted, int count, const SolverOptions& so, double meas_sigma);
    int pack_results(int count, double digest, double* d_out, void* stream);   // `stream` (cudaStream_t) first waits for the match
    int collect_previous();                                                     // call after the match is known to have completed
    void* stream_handle() const;                                                // cudaStream_t of the engine
    int wait_for_stream(void* other_stream);                                    // `other_stream` waits for everything enqueued on the engine's stream so far
    bool map_update_pending() const { return pending_maps_ != 0; }
    const uint64_t* settled_store_counters() const { return settled_counters_; }   // {allocated, detached, freed, free slots} at the last settle
    const std::vector<HostMapStats>& last_map_stats() const { return last_map_stats_; }

    // Particles dst_first .. dst_first+count-1 become copy-on-write copies of src_particle (same set).
    int share_from(int src_particle, int dst_first, int count);
    // new particle k = old particle idx[k] for all resident slots (PFSlam2D::resample's map copies);
    // idx[k] == -1 leaves slot k empty.
    int resample(const int32_t* idx);
    // Serialise / restore the two maps of one resident slot (particle migration between GPUs).
    // Layout: {u32 magic, u32 dim, u32 n_occ, u32 n_dm} + n x u32 directory index + n patches (4 KiB) + n x 128 B obstacle-mirror bits.
    // Device-side form (NCCL send / recv between GPUs): the blob = n x u32 directory index + n patches + n x 128 B mirror bits stays in a
    // device arena owned by the engine (valid until migration_reset()); counts = {occupancy patches, distance patches}.
    struct DeviceBlob { void* dptr = nullptr; size_t bytes = 0; uint32_t n_occ = 0, n_dm = 0; };
    int pack_device(int particle, DeviceBlob* out);
    int migration_alloc(size_t bytes, void** dptr);           // receive buffer in the same arena
    int unpack_device(int particle, const DeviceBlob& blob, bool check = true);   // check = false: no status read-back / synchronisation (the last call of a batch checks)
    void migration_reset();
    int pack_size(int particle, size_t* bytes);
    int pack(int particle, void* buf, size_t cap, size_t* used);
    int unpack(int particle, const void* buf, size_t bytes);

    // Posed scans cast into particle 0's frequency map (GraphSlam2D::generateOccupancyMap's loop, graph_slam2d.cpp:136-160; needs
    // known_plane): scan k = points [offsets[k], offsets[k + 1]) of pts (xyz), sensor origin / quaternion xyzw origins + 3k / quats + 4k
    // (null: identity), base pose states[k].  Every hit cell gets setOccupied and, with `full`, every interior ray cell setFree;
    // *cells = number of cell updates.
    int render_scans(const double* pts, const int64_t* offsets, int n_scans, const double* origins, const double* quats, const SE2* states, bool full,
                     uint64_t* cells);
    // FrequencyOccupancyMap::prune (frequency_occupancy_map.cpp:149-158) of particle 0's map
    int prune_frequency();

    // Direct DynamicDistanceMap::addObstacle / removeObstacle calls in list order, then update().
    int dm_apply(int particle, const uint32_t* cells_xy, const uint8_t* is_add, int n, uint32_t* processed);
    // Likelihoods of Loc2D::addSamplingCovariance for n offsets (x, y pairs) around `pose` on the current scan.
    int sampling_likelihood(int particle, const SE2& pose, const double* offsets_xy, int n, int stride, double* out);
    // Batched DistanceMap::distance(p, &grad).
    int dm_distance(int particle, const double* pts, int n, double* dist, double* grad);

    // Dense window export of raw cell words (kind 0 = occupancy, 1 = distance); present may be null.
    int export_window(int particle, int kind, uint32_t x0, uint32_t y0, int w, int h, uint32_t* words, uint8_t* present);
    int import_window(int particle, int kind, uint32_t x0, uint32_t y0, int w, int h, const uint32_t* words);
    // dense window of a bit plane of the occupancy map: 0 = obstacle mirror, 1 = known bits (log-odds maps)
    int export_bits(int particle, int plane, uint32_t x0, uint32_t y0, int w, int h, uint8_t* out);
    // raw words of n scattered cells (x, y pairs) of one map; flags bit 0: patch exists, bit 1: known bit of a log-odds map
    int gather_cells(int particle, int kind, const uint32_t* cells_xy, int n, uint32_t* words, uint8_t* flags);
    // bounding box (in cells) of allocated patches of one map; returns the number of patches
    int bounds(int particle, int kind, uint32_t mn[2], uint32_t mx[2]);
    // Map::memory() (src/sdm/map.cpp:115-125) of one map kind of every particle: per patch 72 bytes of table entry (key, COWPtr = shared_ptr + mutex, pointer)
    // plus the container's cell bytes divided by its use count; out[particle] truncated to an integer like the reference's return value
    int memory_usage(int kind, uint32_t cell_bytes, uint64_t* out);

    // Checkpoints.  snapshot() settles, checks that every slot's reference count equals its directory references (LAMA_ERR_STATE when
    // not), and copies the slots in use, renumbered, with the directories of the current set into `out`; the engine is not changed.
    // restore() creates an engine with the image's geometry and window on `device` / `stream`: the K slots become 0 .. K-1, the
    // directories set 0, the free stack holds K .. n_slots-1 with the lowest on top (as a fresh engine).  The image must be valid
    // (checkpoint.h checks it).
    int snapshot(EngineImage* out, CheckpointTimes* t = nullptr);
    static Engine* restore(const EngineImage& img, int device, uint64_t stream, std::string& err, CheckpointTimes* t = nullptr);
    // config().center_x / center_y: the world position the window was created around.  The image holds the window base, not the
    // centre, so a restored engine reports (0, 0) until a front end that places other maps on that centre sets it back.
    void set_center(double x, double y) { cfg_.center_x = x; cfg_.center_y = y; }

    // sticky device error bits (lama_core.h) -- reads the device word; 0 = ok
    uint32_t device_status();
    // {patches allocated, patches detached (COW copies), patches freed, free slots}
    void store_counters(uint64_t out[4]);

    void enable_timing(bool on) { timing_ = on; }
    KernelTimes times() const { return times_; }
    void reset_times() { times_ = KernelTimes(); }
    int synchronize();
    uint64_t h2d_bytes() const { return h2d_bytes_; }
    uint64_t d2h_bytes() const { return d2h_bytes_; }
    void reset_traffic() { h2d_bytes_ = d2h_bytes_ = 0; }

    DirWindow window() const { return window_; }

    struct Impl;

private:
    Engine() = default;
    Impl* d_ = nullptr;
    int ensure_states(int count);
    EngineConfig cfg_;
    DirWindow window_{};
    uint32_t max_sqdist_ = 0;
    bool lo_ray_ = false;
    int cur_set_         = 0;
    bool timing_         = false;
    KernelTimes times_;
    std::string err_;
    uint64_t h2d_bytes_ = 0, d2h_bytes_ = 0;
    int pending_maps_ = 0;
    int pending_buf_ = 0;                 // which half of the ping-pong host buffers the pending map update reports into
    uint64_t settled_counters_[4] = {0, 0, 0, 0};
    std::vector<HostMapStats> last_map_stats_;
    bool enq_had_pending_ = false;        // step_enqueue: the previous scan's map update still has to be booked (collect_previous)
    int enq_prev_count_ = 0, enq_prev_buf_ = 0;
    void set_moving(const double origin[3], const double quat[4], double truncated_ray, double truncated_range, int n);
    int enqueue_report(int count);
    int fail(const std::string& what, int code);
    int check_device_status();
};

// error codes returned through the C-ABI
enum : int {
    LAMA_OK            = 0,
    LAMA_ERR_ARG       = -1,
    LAMA_ERR_CUDA      = -2,
    LAMA_ERR_NO_DEVICE = -3,
    LAMA_ERR_WINDOW    = -4,   // the map grew outside the directory window
    LAMA_ERR_POOL      = -5,   // patch pool exhausted
    LAMA_ERR_OVERFLOW  = -6,   // event log / heap / push-list overflow
    LAMA_ERR_STATE     = -7,
};

// Translation3d(origin) * Quaterniond(quat xyzw) of a PointCloudXYZ (types.h:111-120); NULL = zero / identity
MovingTf moving_tf(const double origin[3], const double quat[4]);

}  // namespace lama_b200
