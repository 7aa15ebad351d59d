// kernels.cuh -- launch interface of the sm_90a kernels (implemented in kernels.cu).
#pragma once

#include <cuda_runtime.h>

#include "device_store.cuh"
#include "match_core.h"
#include "ray_core.h"
#include "ray_pull.h"

namespace lama_b200 {

struct MatchResult {
    SE2 state;                 // final state (mode 0) or the evaluated state (mode 1)
    double sums[kNumSums];     // weighted normal equations, chi2, sum d^2, likelihood at `state`
    uint32_t iterations;       // Solver iterations performed
    uint32_t evals_ref;        // residual evaluations the reference's loop performs for this solve
    uint32_t evals_done;       // residual evaluations this kernel actually performed
    uint32_t pad;
};

struct MatchParams {
    const double* points;  // device, N x 3
    ScanParams scan;
    SolverOptions solver;
    double meas_sigma;
    double resolution;
    uint32_t max_sqdist;
    int set;
    int particle_offset;   // particle handled by block 0
    int shared_map;        // 1: every block reads particle `particle_offset`'s map (pose batches on one map)
    int mode;              // 0 = solve + final evaluation, 1 = single evaluation at the input state
};

// per-particle output of k_ray_setup, input of k_ray_pull (the pull form of the ray cast, ray_pull.h)
struct RayPullHeader {   // 64 bytes
    int32_t ox, oy;       // window-relative origin cell of the scan
    int32_t prefix[9];    // class c of the slope-sorted beam list = [prefix[c], prefix[c + 1])
    int32_t n_hits;
    int32_t ok;           // 1: this particle's scan goes through k_ray_pull; 0: k_raycast handles it (tilted sensor, truncated rays)
    int32_t task_base, n_tasks;   // this particle's patches in RayPullView::tasks
    int32_t pad;
};
struct RayPullView {
    RayPullHeader* hdr;   // [particles]
    PullEntry* list;      // [particles][stride]  class lists sorted by (class, slope, beam)
    uint32_t* hits;       // [particles][stride]  pull_hit_record, grouped by patch
    uint2* tasks;         // [particles * dir_dim^2]  {particle << 16 | directory index, first hit record << 16 | number of hit records}
    int32_t* ctrl;        // [0] tasks appended by k_ray_setup, [1] work units taken by k_ray_pull (both reset by k_merge_free)
    int32_t stride;
    int32_t splits;       // work units per particle (a unit = every splits-th patch of one particle)
};

struct RayParams {
    const double* points;
    ScanParams scan;
    int set;
    int particle_offset;
    int state_stride;        // bytes between the poses handed to k_raycast (sizeof(SE2), or sizeof(MatchResult) when it reads k_match's output)
    int log_cap, event_cap;  // powers of two
    int cand_cap;            // candidate bitmaps (patches with hit cells or distance-map obstacles), <= 253
    int debug;               // developer experiments (LAMA_RAY_DEBUG, only honoured by LAMA_PHASE_TIMING builds): 1 no RED, 2 no LDS,
                             // 4 no RED in the walk of x-major beam groups, 8 no RED in the walk of y-major beam groups
    int prob_mode;           // 1: log-odds occupancy (ProbabilisticOccupancyMap), counts go to the scratch map first
    int pull_fallback;       // 1: k_raycast only handles the particles k_ray_setup left to it (RayPullHeader::ok == 0)
    ProbParams prob;
    RayPullView pull;
};

struct BrushParams {
    int set;
    int particle_offset;
    int event_cap;         // stride of the per-particle event lists
    int lower_cap, raise_cap;
    uint32_t max_sqdist;
    int debug;             // LAMA_PHASE_TIMING builds only: print the per-particle phase cycles of this launch
};

// per-particle outputs of the map update
struct MapUpdateStats {
    uint32_t ray_cells;    // cells touched by the ray cast incl. hit cells (work counter C)
    uint32_t log_records;  // touches that needed ordered replay
    uint32_t events;       // effective addObstacle/removeObstacle calls
    uint32_t dm_pops;      // DynamicDistanceMap::update() return value (work counter W)
};

size_t match_smem_bytes(int dir_dim, uint32_t max_sqdist);
size_t raycast_smem_bytes(int dir_dim, const RayParams& rp);
size_t brushfire_smem_bytes(int dir_dim, const BrushParams& bp);
cudaError_t configure_kernels(int dir_dim, uint32_t max_sqdist_limit, const RayParams& rp, const BrushParams& bp);

void launch_match(const StoreView& s, const MatchParams& mp, const SE2* d_states, MatchResult* d_results, int count, cudaStream_t st);
void launch_raycast(const StoreView& s, const RayParams& rp, const SE2* d_states, uint64_t* d_events, MapUpdateStats* d_stats, int count,
                    cudaStream_t st);
// the pull form (every beam planar and starting in the same cell): k_ray_setup + k_ray_pull; particles it cannot take are left to
// launch_raycast with rp.pull_fallback = 1
size_t ray_setup_smem_bytes(int dir_dim, int n_beams);
size_t ray_pull_smem_bytes(int n_beams);
void launch_raycast_pull(const StoreView& s, const RayParams& rp, const SE2* d_states, uint64_t* d_events, MapUpdateStats* d_stats, int count, int n_sms,
                         cudaStream_t st);
void launch_brushfire(const StoreView& s, const BrushParams& bp, uint64_t* d_events, MapUpdateStats* d_stats, int count, cudaStream_t st);
// dst_set[dst_first + k] = src_set[idx[k]] for k in [0, count); bumps reference counts (COW share)
void launch_copy_dirs(const StoreView& s, int src_set, int dst_set, const int32_t* d_idx, int dst_first, int count, cudaStream_t st);
// releases every patch referenced by particles [first, first+count) of `set` and clears their directories
void launch_release(const StoreView& s, int set, int first, int count, cudaStream_t st);
void launch_merge_free(const StoreView& s, cudaStream_t st);
// sharded exchange: kShardFields doubles per particle out of the match results (state, likelihood, evaluation / iteration counts) + one digest
constexpr int kShardFields = 7;
void launch_pack_results(const MatchResult* d_results, int n, double digest, double* d_out, cudaStream_t st);
void launch_gather_cells(const StoreView& s, int set, int particle, int kind, const uint32_t* d_cells, int n, uint32_t* d_words, uint8_t* d_flags,
                         cudaStream_t st);
void launch_delete_patches(const StoreView& s, int set, int particle, const int32_t* d_list, int count, cudaStream_t st);
void launch_init_store(const StoreView& s, int n_sets, cudaStream_t st);
// dense window of one bit plane (0 = obstacle mirror, 1 = known bits of log-odds maps) of an occupancy map, one byte per cell
void launch_export_bits(const StoreView& s, int plane, int set, int particle, uint32_t x0, uint32_t y0, int w, int h, uint8_t* d_out, cudaStream_t st);
// dense window export: out[j * w + i] = cell word or 0; present[..] = 1 when the patch exists
void launch_export(const StoreView& s, int set, int particle, int kind, uint32_t x0, uint32_t y0, int w, int h, uint32_t* d_out,
                   uint8_t* d_present, cudaStream_t st);
// dense, patch-aligned window import (x0,y0 multiples of 32; w,h multiples of 32); all-zero patches are skipped
void launch_import(const StoreView& s, int set, int particle, int kind, uint32_t x0, uint32_t y0, int w, int h, const uint32_t* d_in,
                   cudaStream_t st);
// one warp per listed slot: 4 KiB of cells to d_out, 128 B of obstacle-mirror bits to d_out_fbits and, when d_out_kbits is not null and the
// store has a known plane, 128 B of known bits to d_out_kbits
void launch_gather_patches(const StoreView& s, const int32_t* d_slots, int n, uint32_t* d_out, uint32_t* d_out_fbits, uint32_t* d_out_kbits,
                           cudaStream_t st);
// device scratch of a checkpoint snapshot: cnt / used / new_id / list / ref are n_slots entries, dirs the directories of one set
struct CkptScratch {
    int32_t *cnt, *used, *new_id, *list, *ref, *dirs;
    uint32_t* bad;      // bit 0: a directory entry points outside the pool, bit 1: a reference count differs from the directory references
    void* temp;         // CUB scan temporary storage
    size_t temp_bytes;
};
size_t ckpt_scan_temp_bytes(int n_slots);
// k_ckpt_count (cnt must be zero) -> [after_count recorded] -> k_ckpt_mark -> exclusive scan of `used` -> k_ckpt_list -> k_ckpt_remap;
// the used slots in ascending order get the ids 0 .. K-1, K = new_id[n_slots - 1] + used[n_slots - 1]
void launch_ckpt_compact(const StoreView& s, int set, const CkptScratch& c, cudaStream_t st, cudaEvent_t after_count);
void launch_scatter_patches(const StoreView& s, int set, int particle, int kind, const int32_t* d_entries, int n, const uint32_t* d_in,
                            const uint32_t* d_in_fbits, cudaStream_t st);
// Loc2D::addSamplingCovariance likelihoods: out[i] for offset i (offsets = n x 2 doubles)
void launch_sampling(const StoreView& s, int set, int particle, const double* d_points, const ScanParams& scan, const SE2& pose, const double* d_offsets,
                     int n_offsets, int stride, double resolution, uint32_t max_sqdist, double* d_out, cudaStream_t st);
// MatchSurface2D::error() of `count` states (block k on the map of particle0 + k, or all on particle0's with shared_map)
void launch_match_error(const StoreView& s, int set, int particle0, bool shared_map, const double* d_points, const ScanParams& scan, const SE2* d_states, int count,
                        double resolution, uint32_t max_sqdist, double* d_out, cudaStream_t st);
// batched DistanceMap::distance(point, &grad) on one particle's distance map (SDM grid interface)
void launch_distance(const StoreView& s, int set, int particle, const double* d_pts, int n, double resolution, uint32_t max_sqdist, double* d_dist,
                     double* d_grad, cudaStream_t st);

// GraphSlam2D::generateOccupancyMap's cast of posed scans into particle 0's frequency map (the map needs the `known` plane)
struct RenderParams {
    const double* points;       // xyz of all scans
    const int64_t* offsets;     // [n_scans + 1]: the points of scan k are [offsets[k], offsets[k + 1])
    const MovingTf* moving;     // [n_scans] sensor pose in the base frame
    const SE2* states;          // [n_scans] base pose
    double scale;               // 1 / resolution
    int full;                   // 1: hits and free rays, 0: hits only
    uint8_t* marks;             // [dim^2] zero on entry, zero again on exit
    unsigned long long* cells;  // += cell updates (hits + ray cells)
};
// mark pass -> allocation of the marked patches -> counting pass -> known bits of the touched patches
void launch_render_scans(const StoreView& s, int set, const RenderParams& p, int n_scans, cudaStream_t st);
// FrequencyOccupancyMap::prune over the whole map of particle 0
void launch_prune_freq(const StoreView& s, int set, cudaStream_t st);

}  // namespace lama_b200
