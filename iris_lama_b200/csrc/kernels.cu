// kernels.cu -- the hand-written sm_90a kernels of the LaMa particle-filter hot path.
//
//   k_match      one CTA per particle: the whole Gauss-Newton / LM scan-matching loop
//                (MatchSurface2D::eval + Solver::solve + GaussNewton, see match_core.h)
//   k_raycast    one CTA per particle: beam ray-cast into the frequency occupancy map with packed
//                atomics + ordered replay of threshold crossings (see ray_core.h)
//   k_brushfire  one warp per particle: DynamicDistanceMap::update() in exact heap order (ddm_core.h)
//   k_copy_dirs / k_release / k_merge_free   resampling = directory copies with COW reference counts
//   k_ckpt_*     checkpoints: reference counts checked, used slots compacted, directories renumbered
//
// All of them are memory/latency bound integer + fp64 work: no tensor cores.  Directories are staged
// into shared memory with TMA bulk copies (cp.async.bulk + mbarrier).
#include "kernels.cuh"

#include <algorithm>
#include <cstdio>

#include <cub/device/device_scan.cuh>

#include "brushfire_warp.cuh"

namespace lama_b200 {

namespace {

constexpr int kMatchThreads = 576;  // upper bound; the launch picks the block size that splits the beams into equal rounds
constexpr int kRayThreads   = 512;  // 2 CTAs/SM at 64 registers (no spills in the walk loop); the kernel is bound by integer issue rate

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ==================================================================================================
// k_match
// ==================================================================================================
struct MatchShared {
    uint64_t bar;
    Affine tf;
    SE2 state;
    SolverControl ctl;
    double sums[kNumSums];
    int done;
    uint32_t evals_done;
};

// metric distance of one cell: DynamicDistanceMap::distance(Vector3ui) (dynamic_distance_map.cpp:140-147)
__device__ __forceinline__ double cell_distance(const uint32_t* __restrict__ pool, const int32_t* dir, const DirWindow& win, uint32_t x, uint32_t y,
                                                const double* dtab, uint32_t max_sqdist)
{
    int di = dir_index(win, x, y);
    if (di < 0) return dtab[max_sqdist];
    int slot = dir[di];
    if (slot < 0) return dtab[max_sqdist];
    uint32_t w = __ldg(pool + (size_t)(slot & kDirSlotMask) * kPatchCells + cell_index(x, y));
    return (w & kDmValid) ? dtab[dm_sqdist(w)] : dtab[max_sqdist];
}

__device__ __forceinline__ void eval_beam(double s[kNumSums], const Affine& tf, const double* __restrict__ pt, double scale,
                                          const uint32_t* __restrict__ pool, const int32_t* dir, const DirWindow& win, const double* dtab,
                                          uint32_t max_sqdist, const SolverOptions& so, double meas_sigma)
{
    double hit[3];
    apply_tf(tf, __ldg(pt), __ldg(pt + 1), __ldg(pt + 2), hit);
    // hit.z is forced to 0 by eval (match_surface_2d.cpp:71); z never enters the 2-D lookup.
    const double mx = w2m_nocast(hit[0], scale), my = w2m_nocast(hit[1], scale);
    const uint32_t dx = (uint32_t)mx, dy = (uint32_t)my;
    const double mu0 = add_rn(mx, -(double)dx), mu1 = add_rn(my, -(double)dy);
    double v[4];
    if ((dx & (kPatchLen - 1)) != kPatchLen - 1 && (dy & (kPatchLen - 1)) != kPatchLen - 1) {
        // all four stencil cells live in one patch: one directory lookup
        const double dmax = dtab[max_sqdist];
        int di = dir_index(win, dx, dy);
        int slot = di < 0 ? -1 : dir[di];
        if (slot < 0) {
            v[0] = v[1] = v[2] = v[3] = dmax;
        } else {
            const uint32_t* p = pool + (size_t)(slot & kDirSlotMask) * kPatchCells + cell_index(dx, dy);
            uint32_t w0 = __ldg(p), w1 = __ldg(p + 1), w2 = __ldg(p + kPatchLen), w3 = __ldg(p + kPatchLen + 1);
            v[0] = (w0 & kDmValid) ? dtab[dm_sqdist(w0)] : dmax;
            v[1] = (w1 & kDmValid) ? dtab[dm_sqdist(w1)] : dmax;
            v[2] = (w2 & kDmValid) ? dtab[dm_sqdist(w2)] : dmax;
            v[3] = (w3 & kDmValid) ? dtab[dm_sqdist(w3)] : dmax;
        }
    } else {
        v[0] = cell_distance(pool, dir, win, dx, dy, dtab, max_sqdist);
        v[1] = cell_distance(pool, dir, win, dx + 1, dy, dtab, max_sqdist);
        v[2] = cell_distance(pool, dir, win, dx, dy + 1, dtab, max_sqdist);
        v[3] = cell_distance(pool, dir, win, dx + 1, dy + 1, dtab, max_sqdist);
    }
    BeamEval e = bilinear(v, mu0, mu1, scale, hit[0], hit[1]);
    accumulate(s, e, so.robust_kind, so.robust_param, meas_sigma);
}

__global__ void __launch_bounds__(kMatchThreads, 2)
k_match(StoreView s, MatchParams mp, const SE2* __restrict__ states_in, MatchResult* __restrict__ results)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int dim2      = s.window.dim * s.window.dim;
    int32_t* dir        = reinterpret_cast<int32_t*>(smem_raw);
    double* dtab        = reinterpret_cast<double*>(smem_raw + (size_t)dim2 * 4);
    MatchShared& sh     = *reinterpret_cast<MatchShared*>(smem_raw + (size_t)dim2 * 4 + (size_t)(mp.max_sqdist + 1) * 8);
    double* part        = reinterpret_cast<double*>(smem_raw + (size_t)dim2 * 4 + (size_t)(mp.max_sqdist + 1) * 8 + ((sizeof(MatchShared) + 15) & ~(size_t)15));
    const int tid       = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int particle  = mp.shared_map ? mp.particle_offset : mp.particle_offset + blockIdx.x;
    const int32_t* gdir = dir_of(s, mp.set, particle, kMapDm);

    if (tid == 0) {
        mbar_init(&sh.bar, 1);
        sh.state = states_in[blockIdx.x];
        sh.ctl.begin(mp.solver);
        sh.done       = 0;
        sh.evals_done = 0;
    }
    // sqrt(sqdist) * resolution for every representable squared distance (same expression as
    // dynamic_distance_map.cpp:143-146, so table entries are bit-identical to the reference's values)
    for (uint32_t k = tid; k <= mp.max_sqdist; k += blockDim.x) dtab[k] = mul_rn(sqrt((double)k), mp.resolution);
    __syncthreads();
    block_stage_tma(dir, gdir, (uint32_t)dim2 * 4u, &sh.bar, 0);

    const int n = mp.scan.n_beams;
    const bool single = mp.mode == 1;
    if (tid == 0) sh.tf = compose_tf_fast(sh.state, mp.scan.moving);
    __syncthreads();
    for (;;) {
        double acc[kNumSums];
#pragma unroll
        for (int k = 0; k < kNumSums; ++k) acc[k] = 0.0;
        const Affine tf = sh.tf;
        for (int b = tid; b < n; b += blockDim.x)
            eval_beam(acc, tf, mp.points + 3 * (size_t)b, mp.scan.scale, s.pool, dir, s.window, dtab, mp.max_sqdist, mp.solver, mp.meas_sigma);
        // Block reduction through shared memory, fixed order (deterministic): every thread parks its 12 partial sums, then warp k adds
        // up sum k over all threads (a strided pass + one warp shuffle tree) -- 12 stores per thread instead of 60 shuffles per value.
#pragma unroll
        for (int k = 0; k < kNumSums; ++k) part[k * kMatchThreads + tid] = acc[k];
        __syncthreads();
        for (int k = warp; k < kNumSums; k += (int)(blockDim.x >> 5)) {
            double v = 0.0;
            for (int t = lane; t < (int)blockDim.x; t += 32) v += part[k * kMatchThreads + t];
            v = warp_sum(v);
            if (lane == 0) sh.sums[k] = v;
        }
        __syncthreads();
        // Solver control on warp 0 (one logical thread; the two transcendental calls of SE2::exp run on two lanes), which also prepares the
        // transform of the next evaluation.
        if (warp == 0) {
            if (lane == 0) {
                ++sh.evals_done;
                if (single || sh.done == 1) {
                    sh.done = 2;  // the evaluation just made is the final one
                } else if (sh.ctl.advance(sh.sums, sh.state)) {
                    // finished.  Unless the last step was reverted, the evaluation just made already is the
                    // one at the final state (likelihood, covariance, rmse); otherwise do one more pass.
                    sh.done = sh.ctl.state_dirty ? 1 : 2;
                }
                if (sh.done != 2) sh.tf = compose_tf_fast(sh.state, mp.scan.moving);
            }
        }
        __syncthreads();
        if (sh.done == 2) break;
    }
    if (tid == 0) {
        MatchResult& r = results[blockIdx.x];
        r.state = sh.state;
        for (int k = 0; k < kNumSums; ++k) r.sums[k] = sh.sums[k];
        r.iterations = sh.ctl.iter;
        r.evals_ref  = sh.ctl.evals_ref;
        r.evals_done = sh.evals_done;
        r.pad        = 0;
    }
}

// ==================================================================================================
// k_raycast
// ==================================================================================================
struct RayShared {
    uint64_t bar;
    Affine tf;
    uint32_t log_count, event_count, cells, err;
    uint32_t work[2];       // work-item counters of the two passes
    uint32_t any_pending, n_cand;
#ifdef LAMA_PHASE_TIMING
    uint32_t walk_cells[2];  // planar walk cells of the first pass in y-major / x-major beam groups
#endif
};

// In-place ascending bitonic sort of n (power of two) 64-bit keys in shared memory by the whole block.
// Compare-exchange distances below 32 stay inside aligned 32-key chunks: a warp keeps a chunk in registers and runs
// those stages with shuffles (no block barrier); only the distances >= 32 go through shared memory with a barrier
// per stage (21 instead of 66 barriers at n = 2048).  Ends with a block barrier.
__device__ __forceinline__ uint64_t bitonic_exchange(uint64_t v, int i, int k, int j)
{
    const uint64_t p = __shfl_xor_sync(0xffffffffu, v, j);
    const bool keep_min = ((i & j) == 0) == ((i & k) == 0);
    return (p < v) == keep_min ? p : v;
}
__device__ __forceinline__ void block_bitonic_sort(uint64_t* a, int n)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    if (n <= 32) {   // one warp, padded with the maximum key
        if (warp == 0 && n > 1) {
            uint64_t v = lane < n ? a[lane] : ~0ull;
            for (int k = 2; k <= 32; k <<= 1)
                for (int j = k >> 1; j > 0; j >>= 1) v = bitonic_exchange(v, lane, k, j);
            if (lane < n) a[lane] = v;
        }
        __syncthreads();
        return;
    }
    // stages k = 2 .. 32 (every distance < 32)
    for (int c = warp; c < n / 32; c += nwarps) {
        const int i = c * 32 + lane;
        uint64_t v = a[i];
        for (int k = 2; k <= 32; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1) v = bitonic_exchange(v, i, k, j);
        a[i] = v;
    }
    __syncthreads();
    for (int k = 64; k <= n; k <<= 1) {
        for (int j = k >> 1; j >= 32; j >>= 1) {
            for (int t = threadIdx.x; t < n / 2; t += blockDim.x) {
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));   // the lower index of pair t
                const uint64_t x = a[i], y = a[i | j];
                if ((x > y) == ((i & k) == 0)) {
                    a[i]     = y;
                    a[i | j] = x;
                }
            }
            __syncthreads();
        }
        for (int c = warp; c < n / 32; c += nwarps) {
            const int i = c * 32 + lane;
            uint64_t v = a[i];
            for (int j = 16; j > 0; j >>= 1) v = bitonic_exchange(v, i, k, j);
            a[i] = v;
        }
        __syncthreads();
    }
}
__device__ __forceinline__ int next_pow2(int v)
{
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

// ---- ray-cast work decomposition ------------------------------------------------------------------------------
// Beams are cached in shared memory as their two end cells.  The interior cells of the planar beams (every 2-D
// scan) are emitted by the 2-axis form of Map::computeRay's integer Bresenham (map.cpp:198-227; with from.z == to.z
// the z axis of the reference's loop never moves: delta_z = 0 and 2 * err_z = 0 < n).  Its state after i steps has
// the closed form   k = floor((2 i d + n) / (2 n)),  coord = from + s k,  err = i d - k n,
// so a walk can start anywhere: work items are (group of 32 adjacent beams, segment of kSegSteps steps), handed to
// warps through a shared counter.  Lanes of a warp walk angularly adjacent beams in lock step (in y-major groups their
// atomics fall into the same sectors; x-major groups walk several steps of fewer beams per instruction, see raycast_pass)
// and every warp gets the same amount of work, whatever the ray lengths.
constexpr int kSegSteps = 64;
// x-major groups: consecutive steps of one beam per reduction instruction (see raycast_pass).  8 = 4 beams x 8 steps; on the H100
// 4 was slower and 16 no faster (DESIGN.md §5)
constexpr int kXStride = 8;
static_assert(32 % kXStride == 0, "the lanes of a warp split evenly over the beams of a round");

struct BeamEnds {      // 16 bytes; WINDOW-RELATIVE cell coordinates (< 2^16)
    uint32_t fx, fy;   // from cell; bit 31 of fx: mark_hit, bit 31 of fy: non-planar (generic 3-axis walk)
    uint32_t tx, ty;   // hit cell
};
constexpr uint32_t kBeamFlag = 0x80000000u;

// The class of a group, decided by the warp that holds its 32 cached beams: x-major when most of its planar beams are (SegWalk::init:
// dx >= dy).  Phase 1a (segment counts) and raycast_pass (segment partition) both decide it here, from the same cache entries.
__device__ __forceinline__ bool group_is_xmajor(const BeamEnds& be)
{
    const bool planar = !(be.fy & kBeamFlag);
    const int adx = abs((int)(be.tx - (be.fx & ~kBeamFlag))), ady = abs((int)(be.ty - (be.fy & ~kBeamFlag)));
    const unsigned planar_lanes = __ballot_sync(0xffffffffu, planar), xmajor_lanes = __ballot_sync(0xffffffffu, planar && adx >= ady);
    return 2 * __popc(xmajor_lanes) > __popc(planar_lanes);
}
// Sector alignment of the strided walk (see raycast_pass): an x-major beam of an x-major group starts segment s >= 1 at step
// s * kSegSteps + 1 - delta (xmajor_seg_shift), so each of its kXStride-step octets covers one aligned 32-byte run of counters along
// its row.  Segment 0 ends at step kSegSteps - delta.  All other beams have delta = 0.
static_assert(kSegSteps % kXStride == 0 && kXStride == 8, "one octet of 4-byte counters = one 32-byte sector");
__device__ __forceinline__ int seg_shift(const BeamEnds& be, bool xgroup)
{
    const uint32_t fx = be.fx & ~kBeamFlag;
    const int adx = abs((int)(be.tx - fx)), ady = abs((int)(be.ty - (be.fy & ~kBeamFlag)));
    return xgroup && !(be.fy & kBeamFlag) && adx >= ady ? xmajor_seg_shift(fx, be.tx) : 0;
}

constexpr uint32_t kCandNone = 0xFF, kCandOverflow = 0xFE;
constexpr uint32_t kInfoSlotMask = 0x00FFFFFFu;   // slot field of a patch-info word; all ones = not writable in this pass

// The inner loop of the ray cast: everything it needs to know about a patch is ONE shared-memory word
//   pinfo[directory index] = [candidate bitmap index : 8][slot the counters go to : 24]
// (slot all ones: the patch cannot be written in this pass), so a step is walk + index + LDS + RED with no
// per-lane patch cache and no divergent lookup.
template <bool kProb>
struct RayCtx {
    const StoreView& s;
    const RayParams& rp;
    const uint32_t* pinfo;
    const uint32_t* cand;      // [cand_cap][32]: bit = cell is a hit cell of this scan or a distance-map obstacle
    uint32_t* pending;         // patches that must be allocated / detached before they can be written
    uint32_t* touched;         // kProb: scratch patches that received counts in this scan
    uint64_t* log;
    RayShared& sh;
    int log2dim;
    bool mark;                 // first pass: note the patches that are not writable yet
    int last_di;               // kProb
#ifdef LAMA_PHASE_TIMING
    bool no_red = false;       // RayParams::debug: skip the reductions of the current touches
#endif

    __device__ __forceinline__ uint32_t dir_of_cell(uint32_t P) const { return packed_dir_index(P, log2dim); }

    // One touch of packed cell P whose patch-info word is `info` (directory entry `di`).  `run` > 0: this lane adds the misses of
    // `run` adjacent lanes that touch the same cell (see raycast_pass); `run` == 0: another lane carries this lane's count, only
    // the ordered-path log is kept.  Every counter update is a fire-and-forget reduction at the L2 (SASS RED): nothing waits
    // for a returned value.
    __device__ __forceinline__ void cell(uint32_t P, uint32_t info, uint32_t di, uint32_t beam, uint32_t pos, bool hit, uint32_t run)
    {
        const uint32_t slot = info & kInfoSlotMask;
        if (slot == kInfoSlotMask) {
            if (mark) atomicOr(&pending[di >> 5], 1u << (di & 31));
            return;
        }
        if (kProb && (int)di != last_di) {
            atomicOr(&touched[di >> 5], 1u << (di & 31));
            last_di = (int)di;
        }
        const uint32_t off = packed_cell_offset(P);   // byte offset of the cell in its patch
        if (run) {
            // the pool is 4 KiB aligned (checked at creation): patch base = pool + slot * 4096, the cell offset is OR-ed in
            uint64_t addr;
            uint32_t lo, hi;
            asm("mad.wide.u32 %0, %1, 4096, %2;" : "=l"(addr) : "r"(slot), "l"(s.pool));
            asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(addr));
            lo |= off;
            asm("mov.b64 %0, {%1, %2};" : "=l"(addr) : "r"(lo), "r"(hi));
#ifdef LAMA_PHASE_TIMING
            if (no_red) { if (addr == 1) sh.err = lo; } else
#endif
            asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(addr), "r"(hit ? kOccHitInc : run * kOccMissInc) : "memory");
        }
        if (info >= (kCandNone << 24)) return;   // no candidate cell in this patch (the common case): one compare on the whole word
        const uint32_t ccand = info >> 24;
        const uint32_t ci = off >> 2;
        if (hit || ccand == kCandOverflow || ((cand[ccand * 32 + (ci >> 5)] >> (ci & 31)) & 1u)) {
            const uint32_t idx = atomicAdd(&sh.log_count, 1u);
            if (idx < (uint32_t)rp.log_cap) log[idx] = log_record(P, beam, hit ? 0u : pos, hit);
        }
    }
    // All cells of a beam lie inside the bounding box of its end cells, which phase 1a checked against the window.
    __device__ __forceinline__ void touch(uint32_t P, uint32_t beam, uint32_t pos, bool hit, uint32_t run = 1u)
    {
        const uint32_t di = dir_of_cell(P);
#ifdef LAMA_PHASE_TIMING
        const uint32_t info = (rp.debug & 2) ? (0xFF000000u | (di & 1023u)) : pinfo[di];
#else
        const uint32_t info = pinfo[di];
#endif
        cell(P, info, di, beam, pos, hit, run);
    }
};

// One pass over all touches of the scan (hits, planar segments, generic beams).
template <bool kProb>
__device__ __forceinline__ void raycast_pass(RayCtx<kProb>& c, const BeamEnds* beams, const uint32_t* seg_prefix, int n_beams, int n_groups, uint32_t* work_counter,
                                             const double* __restrict__ points, const Affine& tf, uint32_t bx0, uint32_t by0)
{
    const int tid = threadIdx.x, lane = tid & 31;
    c.last_di = -1;
#ifdef LAMA_PHASE_TIMING
    c.no_red = c.rp.debug & 1;
#endif
    // hits (setOccupied, pf_slam2d.cpp:493-498)
    for (int b = tid; b < n_beams; b += blockDim.x) {
        const BeamEnds be = beams[b];
        if (be.fx & kBeamFlag) c.touch(be.tx | (be.ty << 16), (uint32_t)b, 0u, true);
    }
    // planar beams: warp-dynamic (group, segment) items
    const uint32_t total = seg_prefix[n_groups];
    for (;;) {
        uint32_t item = 0;
        if (lane == 0) item = atomicAdd(work_counter, 1u);
        item = __shfl_sync(0xffffffffu, item, 0);
        if (item >= total) break;
        // group of the item: number of groups whose segment range ends at or before it (<= 128 groups)
        int g = 0;
        for (int g0 = 0; g0 < n_groups; g0 += 32) {
            const int gi = g0 + lane;
            g += __popc(__ballot_sync(0xffffffffu, gi < n_groups && seg_prefix[gi + 1] <= item));
        }
        const int seg = (int)(item - seg_prefix[g]);
        const int b = g * 32 + lane;
        const BeamEnds be = beams[b];   // the cache is padded to whole groups (padding lanes are flagged non-planar)
        const bool planar = !(be.fy & kBeamFlag);
        const bool xgroup = group_is_xmajor(be);
        const int shift = seg_shift(be, xgroup);
#ifdef LAMA_PHASE_TIMING
        c.no_red = (c.rp.debug & 1) || (c.rp.debug & (xgroup ? 4 : 8));
        const int adx = abs((int)(be.tx - (be.fx & ~kBeamFlag))), ady = abs((int)(be.ty - (be.fy & ~kBeamFlag)));
        const int seg_cells = planar ? min(max(adx, ady) - 1, (seg + 1) * kSegSteps - shift) - max(seg * kSegSteps - shift, 0) : 0;
        const uint32_t cells = __reduce_add_sync(0xffffffffu, (uint32_t)max(seg_cells, 0));
        if (c.mark && lane == 0) atomicAdd(&c.sh.walk_cells[xgroup], cells);
#endif
        if (seg == 0 || !xgroup) {
            // Issue order of segment 0 and of y-major groups: lane = beam, one step at a time.  In a y-major group the lanes of one step
            // share a row, so one reduction instruction falls into a few sectors.  Lanes walk angularly adjacent beams in lock step, so
            // neighbouring lanes often sit on the same cell (everywhere close to the sensor, in y-major groups for several segments):
            // runs of equal cells are merged into ONE reduction carrying the run length (counter additions commute; the visited
            // half-word wraps like the reference's uint16).  The ordered-path log stays per touch.
            const int i0 = max(seg * kSegSteps - shift, 0);
            SegWalk w;
            w.init(be.fx & ~kBeamFlag, be.fy & ~kBeamFlag, be.tx, be.ty, i0, planar ? (seg + 1) * kSegSteps - shift - i0 : 0);
            for (;;) {
                const bool v = w.next();
                const unsigned valid = __ballot_sync(0xffffffffu, v);
                if (!valid) break;
                const uint32_t pkey = __shfl_up_sync(0xffffffffu, w.P, 1);
                const bool head = v && (lane == 0 || !((valid >> (lane - 1)) & 1u) || pkey != w.P);
                const unsigned heads = __ballot_sync(0xffffffffu, head);
                if (v) {
                    const unsigned stop = (heads | ~valid) & ~((2u << lane) - 1u);   // first lane above that starts another run
                    const uint32_t run = head ? (uint32_t)((stop ? __ffs(stop) - 1 : 32) - lane) : 0u;
                    c.touch(w.P, (uint32_t)b, (uint32_t)w.i, false, run);
                }
            }
        } else {
            // Issue order of the later segments of an x-major group.  The lanes of one step share a COLUMN (up to 32 lines), so
            // kXStride lanes walk one beam at consecutive offsets with stride kXStride: one instruction covers 32 / kXStride beams x
            // kXStride consecutive steps along their rows, and the group's beams take kXStride rounds.  The segments of x-major beams
            // are shifted back by seg_shift, so those kXStride cells of a beam fill one 32-byte sector whenever the minor axis does not
            // move among them.  The cells touched are the same (counter additions commute, the log is sorted), only the order of the
            // reductions changes.
            for (int round = 0; round < kXStride; ++round) {
                const int bb = g * 32 + round * (32 / kXStride) + lane / kXStride;
                const BeamEnds e = beams[bb];
                const int first = seg * kSegSteps + 1 - seg_shift(e, true);
                StrideWalk sw;
                sw.init(e.fx & ~kBeamFlag, e.fy & ~kBeamFlag, e.tx, e.ty, first + lane % kXStride,
                        (e.fy & kBeamFlag) ? 0 : first + kSegSteps - 1, kXStride);
                if (sw.i > sw.iend) continue;
                // software pipeline: the patch-info word of the NEXT cell is fetched from shared memory before the current cell is
                // processed, so the load latency overlaps the address arithmetic and the reduction of the current cell.  The walk never
                // steps past the lane's last cell, so every directory index it forms lies inside the beam's bounding box.
                uint32_t P = sw.P, di = c.dir_of_cell(P);
                uint32_t info = c.pinfo[di];
                const int last_prefetch = sw.iend - kXStride;
                while (sw.i <= last_prefetch) {
                    const uint32_t pos = (uint32_t)sw.i;
                    sw.step();
                    const uint32_t Pn = sw.P, din = c.dir_of_cell(Pn);
                    const uint32_t infon = c.pinfo[din];
                    c.cell(P, info, di, (uint32_t)bb, pos, false, 1u);
                    P = Pn; di = din; info = infon;
                }
                c.cell(P, info, di, (uint32_t)bb, (uint32_t)sw.i, false, 1u);
            }
        }
    }
#ifdef LAMA_PHASE_TIMING
    c.no_red = c.rp.debug & 1;
#endif
    // non-planar beams (tilted sensor): the reference's 3-axis walk, one thread per beam
    for (int b = tid; b < n_beams; b += blockDim.x) {
        if (!(beams[b].fy & kBeamFlag)) continue;
        const double pt[3] = {__ldg(points + 3 * (size_t)b), __ldg(points + 3 * (size_t)b + 1), __ldg(points + 3 * (size_t)b + 2)};
        const BeamCells bc = beam_cells(tf, c.rp.scan, pt);
        RayWalk3 w(bc);
        while (w.next()) c.touch((w.x - bx0) | ((w.y - by0) << 16), (uint32_t)b, (uint32_t)w.i, false);
    }
}

// kProb = false: FrequencyOccupancyMap (PFSlam2D / Slam2D); kProb = true: ProbabilisticOccupancyMap -- the walk adds
// the per-scan {hits, touches} into a scratch map, candidate cells are replayed in order on the float cell, all other
// touched cells (misses only, never an obstacle) get their k misses applied one by one in a bulk pass.
#ifdef LAMA_PHASE_TIMING   // developer build: per-phase cycle counts of two CTAs (make EXTRA=-DLAMA_PHASE_TIMING)
#define RAY_MARK(k) do { if (tid == 0 && (blockIdx.x == 0 || blockIdx.x == 200)) ph[k] = clock64(); } while (0)
#else
#define RAY_MARK(k) do { } while (0)
#endif

template <bool kProb>
__global__ void __launch_bounds__(kRayThreads, kProb ? 1 : 2)
k_raycast(StoreView s, RayParams rp, const SE2* __restrict__ states, uint64_t* __restrict__ events_out, MapUpdateStats* __restrict__ stats)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int dim2   = s.window.dim * s.window.dim;
    const int nwords = (dim2 + 31) / 32;
    const int n      = rp.scan.n_beams;
    const int n_groups = (n + 31) / 32;
    int32_t* dir     = reinterpret_cast<int32_t*>(smem_raw);
    uint64_t* log    = reinterpret_cast<uint64_t*>(smem_raw + (size_t)dim2 * 4);
    BeamEnds* beams  = reinterpret_cast<BeamEnds*>(log + rp.log_cap);
    uint64_t* events = reinterpret_cast<uint64_t*>(beams);  // overlays the beam cache, which is dead by then
    const size_t beam_bytes = (size_t)n_groups * 32 * sizeof(BeamEnds), ev_bytes = (size_t)rp.event_cap * 8;
    uint32_t* cand   = reinterpret_cast<uint32_t*>(reinterpret_cast<unsigned char*>(beams) + (beam_bytes > ev_bytes ? beam_bytes : ev_bytes));
    uint32_t* hotmap = cand + rp.cand_cap * 32;
    uint32_t* pending = hotmap + nwords;
    uint32_t* seg_prefix = pending + nwords;           // n_groups + 1 entries
    uint32_t* pinfo  = seg_prefix + ((n_groups + 2) & ~1);   // per directory entry: [candidate bitmap index : 8][slot : 24]
    uint16_t* cand_di = reinterpret_cast<uint16_t*>(pinfo + dim2);  // directory entry of every bitmap
    RayShared& sh    = *reinterpret_cast<RayShared*>(cand_di + ((rp.cand_cap + 3) & ~3));
    const size_t dir_s_off = ((size_t)(reinterpret_cast<unsigned char*>(&sh) - smem_raw) + sizeof(RayShared) + 15) & ~(size_t)15;  // TMA target: 16-B aligned
    int32_t* dir_s   = reinterpret_cast<int32_t*>(smem_raw + dir_s_off);                                                                  // kProb only
    uint32_t* touched = reinterpret_cast<uint32_t*>(dir_s + dim2);                                                                  // kProb only

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    if (rp.pull_fallback && rp.pull.hdr[blockIdx.x].ok) return;   // k_ray_setup / k_ray_pull took this particle's scan
    const int particle = rp.particle_offset + blockIdx.x;
    int32_t* gdir      = dir_of(s, rp.set, particle, kMapOcc);
    int32_t* gdir_s    = kProb ? dir_of(s, rp.set, particle, kMapScratch) : nullptr;
    const DirWindow win = s.window;
    const uint32_t bx0 = (uint32_t)win.base_px << kPatchLog2, by0 = (uint32_t)win.base_py << kPatchLog2;
    const uint32_t side = (uint32_t)win.dim << kPatchLog2;
    int log2dim = 0;
    while ((1 << (log2dim + 1)) <= win.dim) ++log2dim;

#ifdef LAMA_PHASE_TIMING
    long long ph[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
#endif
    RAY_MARK(0);
    // ---- phase 0: stage the directory, clear scratch -------------------------------------------------
    if (tid == 0) {
        mbar_init(&sh.bar, 1);
        sh.tf = compose_tf(*reinterpret_cast<const SE2*>(reinterpret_cast<const char*>(states) + (size_t)blockIdx.x * (size_t)rp.state_stride), rp.scan.moving);
        sh.log_count = sh.event_count = sh.cells = sh.err = 0;
        sh.work[0] = sh.work[1] = 0;
        sh.any_pending = 0;
        sh.n_cand = 0;
#ifdef LAMA_PHASE_TIMING
        sh.walk_cells[0] = sh.walk_cells[1] = 0;
#endif
    }
    for (int i = tid; i < 2 * nwords; i += blockDim.x) hotmap[i] = 0u;  // hotmap + pending are contiguous
    for (int i = tid; i < dim2; i += blockDim.x) pinfo[i] = 0xFFFFFFFFu;  // kCandNone, not writable
    if (kProb)
        for (int i = tid; i < nwords; i += blockDim.x) touched[i] = 0u;
    __syncthreads();
    block_stage_tma(dir, gdir, (uint32_t)dim2 * 4u, &sh.bar, 0);
    if (kProb) block_stage_tma(dir_s, gdir_s, (uint32_t)dim2 * 4u, &sh.bar, 1);
    const Affine tf = sh.tf;

    // ---- phase 1a: beam end cells, segment counts, patches that need the ordered path ---------------------
    uint32_t my_err = 0, my_cells = 0;   // touches of this scan: every beam's hit + its n - 1 interior cells (each applied exactly once)
    for (int di = tid; di < dim2; di += blockDim.x) {
        const int e = dir[di];
        if (e >= 0 && (e & kDirHot)) atomicOr(&hotmap[di >> 5], 1u << (di & 31));  // holds distance-map obstacles
    }
    for (int b = tid; b < n_groups * 32; b += blockDim.x) {
        BeamEnds be{0u, 0u | kBeamFlag, 0u, 0u};  // padding lanes: flagged non-planar, never walked (b >= n)
        int walk = 0;   // interior cells of a planar beam
        if (b < n) {
            const double pt[3] = {__ldg(rp.points + 3 * (size_t)b), __ldg(rp.points + 3 * (size_t)b + 1), __ldg(rp.points + 3 * (size_t)b + 2)};
            const BeamCells bc = beam_cells(tf, rp.scan, pt);
            be.fx = bc.from[0] - bx0; be.fy = bc.from[1] - by0; be.tx = bc.to[0] - bx0; be.ty = bc.to[1] - by0;
            if ((be.fx | be.fy | be.tx | be.ty) >= side) {  // the beam leaves the directory window: reported, nothing is written
                my_err |= kErrWindow;
                be.fx = be.tx = be.fy = be.ty = 0u;
            } else {
                if (bc.mark_hit) {
                    const int di = (int)(((be.ty >> kPatchLog2) << log2dim) | (be.tx >> kPatchLog2));
                    be.fx |= kBeamFlag;
                    atomicOr(&hotmap[di >> 5], 1u << (di & 31));  // holds a hit cell of this scan
                    my_cells += 1;
                }
                const int ddx = (int)(bc.to[0] - bc.from[0]), ddy = (int)(bc.to[1] - bc.from[1]), ddz = (int)(bc.to[2] - bc.from[2]);
                const int nn = max(max(ddx < 0 ? -ddx : ddx, ddy < 0 ? -ddy : ddy), ddz < 0 ? -ddz : ddz);
                my_cells += nn > 1 ? (uint32_t)(nn - 1) : 0u;
                if (ddz != 0) be.fy |= kBeamFlag;
                else walk = nn - 1;
            }
        }
        beams[b] = be;
        // one warp holds one group: steps 1 .. walk in segments shifted back by seg_shift; a group has the segments of its longest beam
        const bool xgroup = group_is_xmajor(be);   // warp-collective: every lane of the warp, before any lane-dependent branch
        int segs = walk > 0 ? (walk + seg_shift(be, xgroup) + kSegSteps - 1) / kSegSteps : 0;
        segs = __reduce_max_sync(0xffffffffu, segs);
        if (lane == 0) seg_prefix[b >> 5] = (uint32_t)segs;
    }
    __syncthreads();
    // ---- phase 1b: one warp numbers the hot patches and scans the segment counts -----------------------------
    if (warp == 0) {
        uint32_t base = 0;
        for (int w0 = 0; w0 < nwords; w0 += 32) {
            const int wi = w0 + lane;
            const uint32_t bits = wi < nwords ? hotmap[wi] : 0u;
            const uint32_t cnt = __popc(bits);
            uint32_t incl = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            uint32_t k = base + incl - cnt;
            uint32_t b2 = bits;
            while (b2) {
                const int bit = __ffs(b2) - 1;
                b2 &= b2 - 1;
                const int di = wi * 32 + bit;
                if (k < (uint32_t)rp.cand_cap) {
                    pinfo[di]  = (k << 24) | kInfoSlotMask;
                    cand_di[k] = (uint16_t)di;
                } else {
                    pinfo[di] = (kCandOverflow << 24) | kInfoSlotMask;
                }
                ++k;
            }
            base += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) {
            sh.n_cand = base < (uint32_t)rp.cand_cap ? base : (uint32_t)rp.cand_cap;
            uint32_t acc = 0;
            for (int g = 0; g < n_groups; ++g) {
                uint32_t v = seg_prefix[g];
                seg_prefix[g] = acc;
                acc += v;
            }
            seg_prefix[n_groups] = acc;
        }
    }
    __syncthreads();
    // ---- phase 1c: candidate bitmaps = obstacle-mirror bits of the patch | hit cells of this scan --------------
    for (int k = warp; k < (int)sh.n_cand; k += nwarps) {
        const int e = dir[cand_di[k]];
        cand[k * 32 + lane] = e >= 0 ? __ldcg(fbits_ptr(s, e & kDirSlotMask) + lane) : 0u;
    }
    __syncthreads();
    for (int b = tid; b < n; b += blockDim.x) {
        const BeamEnds be = beams[b];
        if (!(be.fx & kBeamFlag)) continue;
        const int k = (int)(pinfo[((be.ty >> kPatchLog2) << log2dim) | (be.tx >> kPatchLog2)] >> 24);
        if (k < rp.cand_cap) {
            const uint32_t ci = cell_index(be.tx, be.ty);
            atomicOr(&cand[k * 32 + (ci >> 5)], 1u << (ci & 31));
        }
    }
    // ---- phase 1d: the slot every patch's counters go to in the first pass (patches this particle owns) -------------
    for (int di = tid; di < dim2; di += blockDim.x) {
        int e = dir[di];
        bool writable = e >= 0 && (e & kDirOwn);
        if (kProb) {  // the counts of a log-odds map go to the scratch patch; both patches must be owned
            const int se = dir_s[di];
            writable = writable && se >= 0 && (se & kDirOwn);
            e = se;
        }
        if (writable) pinfo[di] = (pinfo[di] & 0xFF000000u) | (uint32_t)(e & kDirSlotMask);
    }
    __syncthreads();

    RAY_MARK(1);
    // ---- phase 2: optimistic pass -- every patch this particle already owns is written right away;
    // ---- phase 3: allocate / detach the patches that were not writable (Map::get mutable + COW) and redo those ----
    RayCtx<kProb> ctx{s, rp, pinfo, cand, pending, touched, log, sh, log2dim, true, -1};
#pragma unroll 1
    for (int pass = 0; pass < 2; ++pass) {
        if (pass == 1) {
            __syncthreads();
            for (int w32 = warp; w32 < nwords; w32 += nwarps) {
                uint32_t bits = pending[w32];
                if (bits && lane == 0) sh.any_pending = 1;
                while (bits) {
                    const int bit = __ffs(bits) - 1;
                    bits &= bits - 1;
                    if (warp_make_exclusive(s, dir, gdir, w32 * 32 + bit, lane) < 0) my_err |= kErrPoolEmpty;
                    if (kProb && warp_make_exclusive(s, dir_s, gdir_s, w32 * 32 + bit, lane) < 0) my_err |= kErrPoolEmpty;
                }
            }
            __syncthreads();
            if (!sh.any_pending) break;
            // second pass: only the cells of the patches that were pending (the others are done)
            for (int di = tid; di < dim2; di += blockDim.x) {
                uint32_t slot = kInfoSlotMask;
                if ((pending[di >> 5] >> (di & 31)) & 1u) {
                    int e = dir[di];
                    bool writable = e >= 0 && (e & kDirOwn);
                    if (kProb) {
                        const int se = dir_s[di];
                        writable = writable && se >= 0 && (se & kDirOwn);
                        e = se;
                    }
                    if (writable) slot = (uint32_t)(e & kDirSlotMask);   // else: the pool ran dry (reported)
                }
                pinfo[di] = (pinfo[di] & 0xFF000000u) | slot;
            }
            __syncthreads();
            ctx.mark = false;
        }
        raycast_pass(ctx, beams, seg_prefix, n, n_groups, &sh.work[pass], rp.points, tf, bx0, by0);
    }
    my_cells = __reduce_add_sync(0xffffffffu, my_cells);
    if (lane == 0 && my_cells) atomicAdd(&sh.cells, my_cells);
    __threadfence();  // the reductions above must have been performed before the replay reads the counters back
    __syncthreads();

    RAY_MARK(2);
    // ---- phase 4: sort the log by (cell, beam) -------------------------------------------------------------
    uint32_t count = sh.log_count;
    if (count > (uint32_t)rp.log_cap) {
        my_err |= kErrEventLog;
        count = rp.log_cap;
    }
    const int padded = next_pow2((int)count);
    for (int i = count + tid; i < padded; i += blockDim.x) log[i] = ~0ull;
    __syncthreads();
    block_bitonic_sort(log, padded);

    __syncthreads();
    RAY_MARK(3);
    // ---- phase 5: per-cell ordered replay -> obstacle events ----------------------------------------------
    for (int i = tid; i < (int)count; i += blockDim.x) {
        const uint32_t key = log_key(log[i]);
        if (i > 0 && log_key(log[i - 1]) == key) continue;  // not a segment head
        int end = i + 1;
        while (end < (int)count && log_key(log[end]) == key) ++end;
        const uint32_t x = key_x(win, key), y = key_y(win, key);
        const int di = dir_index(win, x, y);
        uint32_t* cell = patch_ptr(s, dir[di] & kDirSlotMask) + cell_index(x, y);
        const uint32_t final_word = __ldcg(cell);
        const uint32_t ci = cell_index(x, y);
        uint32_t* fword = fbits_ptr(s, dir[di] & kDirSlotMask) + (ci >> 5);
        const bool before = (__ldcg(fword) >> (ci & 31)) & 1u;
        auto emit = [&](bool add, uint32_t seq) {
            uint32_t idx = atomicAdd(&sh.event_count, 1u);
            if (idx < (uint32_t)rp.event_cap) events[idx] = push_record((seq << 1) | (add ? 1u : 0u), key);
        };
        bool obstacle = before;
        if (kProb) {
            // the float cell is updated here, touch by touch; the bulk pass must skip it: clear its scratch counter
            const float p = replay_cell_prob(log, i, end, __uint_as_float(final_word), obstacle, rp.prob, emit);
            *cell = __float_as_uint(p);
            patch_ptr(s, dir_s[di] & kDirSlotMask)[ci] = 0u;
            atomicOr(kbits_ptr(s, dir[di] & kDirSlotMask) + (ci >> 5), 1u << (ci & 31));
        } else {
            uint32_t word = final_word;
            obstacle = replay_cell(log, i, end, word, before, emit);
            if (word != final_word) *cell = word;   // the replay is the only writer of a logged cell after the barrier
        }
        if (obstacle != before) {
            if (obstacle) {
                atomicOr(fword, 1u << (ci & 31));
                if (!(dir[di] & kDirHot)) {  // from now on this patch needs the ordered path
                    atomicOr(&dir[di], kDirHot);
                    atomicOr(&gdir[di], kDirHot);
                }
            } else {
                atomicAnd(fword, ~(1u << (ci & 31)));
            }
        }
    }
    __syncthreads();

    // ---- phase 5b (log-odds maps): apply the k misses of every other touched cell, one by one ---------------------
    if (kProb) {
        for (int w32 = 0; w32 < nwords; ++w32) {
            uint32_t bits = touched[w32];
            int ord = 0;
            while (bits) {
                const int bit = __ffs(bits) - 1;
                bits &= bits - 1;
                if ((ord++ % nwarps) != warp) continue;  // patches of this word are dealt round-robin to the warps
                const int di = w32 * 32 + bit;
                uint32_t* occ = patch_ptr(s, dir[di] & kDirSlotMask);
                uint32_t* scr = patch_ptr(s, dir_s[di] & kDirSlotMask);
                uint32_t* kb  = kbits_ptr(s, dir[di] & kDirSlotMask);
                for (int row = 0; row < kPatchLen; ++row) {
                    const int ci = row * kPatchLen + lane;
                    const uint32_t c = __ldcg(scr + ci);
                    if (c) {
                        // not a candidate: no hit in this scan and not an obstacle -> misses only, no event possible
                        float p = __uint_as_float(__ldcg(occ + ci));
                        for (uint32_t k = occ_visited(c); k > 0; --k) p = prob_miss(p, rp.prob);
                        occ[ci] = __float_as_uint(p);
                        scr[ci] = 0u;
                    }
                    const uint32_t known = __ballot_sync(0xffffffffu, c != 0u);
                    if (lane == 0 && known) kb[row] |= known;
                }
            }
        }
        __syncthreads();
    }

    RAY_MARK(4);
    // ---- phase 6: order the events like the reference's call sequence and publish them --------------------
    uint32_t nev = sh.event_count;
    if (nev > (uint32_t)rp.event_cap) {
        my_err |= kErrPushOverflow;
        nev = rp.event_cap;
    }
    const int evpad = next_pow2((int)nev);
    for (int i = nev + tid; i < evpad; i += blockDim.x) events[i] = ~0ull;
    __syncthreads();
    block_bitonic_sort(events, evpad);
    uint64_t* out = events_out + (size_t)blockIdx.x * rp.event_cap;
    for (int i = tid; i < (int)nev; i += blockDim.x) out[i] = events[i];
    my_err = __reduce_or_sync(0xffffffffu, my_err);
    if (lane == 0 && my_err) atomicOr(s.status, my_err);
#ifdef LAMA_PHASE_TIMING
    __syncthreads();
    RAY_MARK(5);
    if (tid == 0 && (blockIdx.x == 0 || blockIdx.x == 200))
        printf("ray cta %d debug %d: setup %lld walk %lld sort %lld replay %lld events %lld | log %u events %u | walk cells y-major %u x-major %u\n", blockIdx.x,
               rp.debug, ph[1] - ph[0], ph[2] - ph[1], ph[3] - ph[2], ph[4] - ph[3], ph[5] - ph[4], sh.log_count, sh.event_count, sh.walk_cells[0], sh.walk_cells[1]);
#endif
    if (tid == 0) {
        MapUpdateStats& st = stats[blockIdx.x];
        st.ray_cells   = sh.cells;
        st.log_records = count;
        st.events      = nev;
        st.dm_pops     = 0;
    }
}


// ==================================================================================================
// pull form of the ray cast (ray_pull.h): k_ray_setup + k_ray_pull
// ==================================================================================================
// k_ray_setup, one CTA per particle: beam end cells -> 8 slope-sorted class lists, the hit records grouped by patch and one task per
// patch the scan can touch, appended to one global task list.  A particle whose beams are not all planar with one common origin
// inside the window is left to k_raycast (header.ok = 0).
// Sorting: a counting sort on (class, top 8 bits of the slope) puts every beam within a few places of its final position (beams
// of a sweep are ~1 bucket apart); odd-even transposition passes then run until one changes nothing, which makes the order exact
// for ANY input (a pathological point cloud just needs more passes).
constexpr int kSetupThreads = 512;
constexpr int kSlopeBuckets = 8 * 256;
struct RaySetupShared {
    Affine tf;
    uint32_t ox, oy, bad, cells;
    int n_list, n_hits, n_hpatch, n_tasks, task_base, swapped;
    int prefix[9];
    uint32_t scan[kSetupThreads / 32];
    uint32_t scan_total;
};

// exclusive prefix sum of one value per thread over the block (two barriers); *total = sum over the block
__device__ __forceinline__ uint32_t block_scan_excl(uint32_t v, uint32_t* warp_sums, uint32_t* total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < nwarps ? warp_sums[lane] : 0u, wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += t;
        }
        if (lane < nwarps) warp_sums[lane] = wi - w;
        if (lane == 31) *total = wi;
    }
    __syncthreads();
    return warp_sums[warp] + incl - v;
}

struct RaySetupLayout {
    size_t keys, sorted, ndb, hrec, marks, hmarks, wpfx, hwpfx, bucket, bfill, hcnt, hfill, sh, total;
    __host__ __device__ RaySetupLayout(int n_beams, int dim2)
    {
        const size_t npad = ((size_t)n_beams + 31) & ~(size_t)31, nwords = ((size_t)dim2 + 31) / 32, nw2 = (nwords + 1) & ~(size_t)1;
        size_t o = 0;
        keys = o;   o += npad * 8;
        sorted = o; o += (npad + 2) * 8;
        ndb = o;    o += npad * 4;
        hrec = o;   o += npad * 4;
        marks = o;  o += nw2 * 4;
        hmarks = o; o += nw2 * 4;
        wpfx = o;   o += nw2 * 4;
        hwpfx = o;  o += nw2 * 4;
        bucket = o; o += (size_t)(kSlopeBuckets + 2) * 4;
        bfill = o;  o += (size_t)kSlopeBuckets * 4;
        hcnt = o;   o += (npad + 2) * 4;
        hfill = o;  o += npad * 4;
        o = (o + 15) & ~(size_t)15;
        sh = o;     o += sizeof(RaySetupShared);
        total = o + 16;
    }
};

__global__ void __launch_bounds__(kSetupThreads)
k_ray_setup(StoreView s, RayParams rp, const SE2* __restrict__ states, MapUpdateStats* __restrict__ stats)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int n = rp.scan.n_beams, npad = (n + 31) & ~31;
    const int dim = s.window.dim, dim2 = dim * dim, nwords = (dim2 + 31) / 32;
    const RaySetupLayout L(n, dim2);
    uint64_t* keys   = reinterpret_cast<uint64_t*>(smem_raw + L.keys);     // sort key of beam b (~0: no interior cells)
    uint64_t* sorted = reinterpret_cast<uint64_t*>(smem_raw + L.sorted);
    uint32_t* ndb    = reinterpret_cast<uint32_t*>(smem_raw + L.ndb);      // n | d << 16 of beam b
    uint32_t* hrec   = reinterpret_cast<uint32_t*>(smem_raw + L.hrec);     // directory index << 10 | cell of beam b's hit (~0: none)
    uint32_t* marks  = reinterpret_cast<uint32_t*>(smem_raw + L.marks);    // patches the scan may touch
    uint32_t* hmarks = reinterpret_cast<uint32_t*>(smem_raw + L.hmarks);   // patches holding hit cells
    uint32_t* wpfx   = reinterpret_cast<uint32_t*>(smem_raw + L.wpfx);     // marked patches before word w
    uint32_t* hwpfx  = reinterpret_cast<uint32_t*>(smem_raw + L.hwpfx);
    uint32_t* bucket = reinterpret_cast<uint32_t*>(smem_raw + L.bucket);   // counting sort: counts, then start offsets
    uint32_t* bfill  = reinterpret_cast<uint32_t*>(smem_raw + L.bfill);
    uint32_t* hcnt   = reinterpret_cast<uint32_t*>(smem_raw + L.hcnt);     // hits per hit patch, then start offsets
    uint32_t* hfill  = reinterpret_cast<uint32_t*>(smem_raw + L.hfill);
    RaySetupShared& sh = *reinterpret_cast<RaySetupShared*>(smem_raw + L.sh);
    const int tid = threadIdx.x, lane = tid & 31;
    const RayPullView& pv = rp.pull;
    RayPullHeader* hdr = pv.hdr + blockIdx.x;
    const uint32_t bx0 = (uint32_t)s.window.base_px << kPatchLog2, by0 = (uint32_t)s.window.base_py << kPatchLog2;
    const uint32_t side = (uint32_t)dim << kPatchLog2;
    int log2dim = 0;
    while ((1 << (log2dim + 1)) <= dim) ++log2dim;

    if (tid == 0) {
        sh.tf = compose_tf(*reinterpret_cast<const SE2*>(reinterpret_cast<const char*>(states) + (size_t)blockIdx.x * (size_t)rp.state_stride), rp.scan.moving);
        // the common ray start: tf.translation (pf_slam2d.cpp:449), not moved by any truncation in this mode
        sh.ox = w2m(sh.tf.t[0], rp.scan.scale) - bx0;
        sh.oy = w2m(sh.tf.t[1], rp.scan.scale) - by0;
        sh.bad = (sh.ox | sh.oy) >= side ? 3u : 0u;
        sh.cells = 0;
        sh.n_list = sh.n_hits = 0;
        for (int c = 0; c < 9; ++c) sh.prefix[c] = 0;
    }
    for (int i = tid; i < nwords; i += blockDim.x) marks[i] = hmarks[i] = 0u;
    for (int i = tid; i < kSlopeBuckets; i += blockDim.x) bucket[i] = 0u;
    for (int i = tid; i < npad + 2; i += blockDim.x) hcnt[i] = 0u;
    for (int i = tid; i < npad; i += blockDim.x) hfill[i] = 0u;
    __syncthreads();
    const Affine tf = sh.tf;
    const uint32_t ox = sh.ox, oy = sh.oy;
    uint32_t my_cells = 0, my_bad = 0;
    for (int b = tid; b < npad; b += blockDim.x) {
        uint64_t key = ~0ull;
        uint32_t nd = 0, hr = ~0u;
        if (b < n && !sh.bad) {
            const double pt[3] = {__ldg(rp.points + 3 * (size_t)b), __ldg(rp.points + 3 * (size_t)b + 1), __ldg(rp.points + 3 * (size_t)b + 2)};
            const BeamCells bc = beam_cells(tf, rp.scan, pt);
            const uint32_t fx = bc.from[0] - bx0, fy = bc.from[1] - by0, tx = bc.to[0] - bx0, ty = bc.to[1] - by0;
            if (bc.from[2] != bc.to[2] || fx != ox || fy != oy || (tx | ty) >= side) {
                my_bad |= (tx | ty) >= side ? 3u : 1u;   // bit 1: the beam leaves the directory window (reported, loud)
            } else {
                const int ex = (int)tx - (int)ox, ey = (int)ty - (int)oy;
                const PullBeam pb = pull_classify(ex, ey);
                if (bc.mark_hit) {
                    const uint32_t di = ((ty >> kPatchLog2) << log2dim) | (tx >> kPatchLog2);
                    hr = (di << 10) | cell_index(tx, ty);
                    atomicOr(&marks[di >> 5], 1u << (di & 31));
                    atomicOr(&hmarks[di >> 5], 1u << (di & 31));
                    my_cells += 1;
                }
                if (pb.n >= 2) {
                    my_cells += pb.n - 1;
                    key = pull_sort_key(pb.cls, pb.n, pb.d, (uint32_t)b);
                    nd  = pull_pack(pb.n, pb.d);
                    uint32_t sb = (uint32_t)((key >> 16) >> 31) & 0x1FFu;   // top bits of the 2^39-scaled slope
                    sb = sb > 255u ? 255u : sb;
                    atomicAdd(&bucket[pb.cls * 256 + (int)sb], 1u);
                    pull_mark_beam(ox, oy, ex, ey, [&](int px, int py) {
                        const uint32_t di = ((uint32_t)py << log2dim) | (uint32_t)px;
                        atomicOr(&marks[di >> 5], 1u << (di & 31));
                    });
                }
            }
        }
        keys[b] = key;
        ndb[b]  = nd;
        hrec[b] = hr;
    }
    my_cells = __reduce_add_sync(0xffffffffu, my_cells);
    my_bad   = __reduce_or_sync(0xffffffffu, my_bad);
    if (lane == 0) {
        if (my_cells) atomicAdd(&sh.cells, my_cells);
        if (my_bad) atomicOr(&sh.bad, my_bad);
    }
    __syncthreads();
    if (sh.bad) {   // not for this path: k_raycast takes the particle
        if (tid == 0) {
            hdr->ok = 0;
            if (sh.bad & 2u) atomicOr(s.status, kErrWindow);
        }
        return;
    }
    // ---- bucket starts; number the marked patches (tasks) and the hit patches ------------------------------------
    {
        constexpr int per = kSlopeBuckets / kSetupThreads;
        uint32_t c[per], sum = 0;
#pragma unroll
        for (int k = 0; k < per; ++k) { c[k] = bucket[tid * per + k]; sum += c[k]; }
        uint32_t base = block_scan_excl(sum, sh.scan, &sh.scan_total);
#pragma unroll
        for (int k = 0; k < per; ++k) { bucket[tid * per + k] = base; bfill[tid * per + k] = base; base += c[k]; }
        if (tid == 0) sh.n_list = (int)sh.scan_total;
        __syncthreads();
        const uint32_t m0 = tid < nwords ? (uint32_t)__popc(marks[tid]) : 0u;   // nwords <= 512 (dir_dim <= 128)
        const uint32_t p0 = block_scan_excl(m0, sh.scan, &sh.scan_total);
        if (tid < nwords) wpfx[tid] = p0;
        if (tid == 0) {
            sh.n_tasks   = (int)sh.scan_total;
            sh.task_base = atomicAdd(pv.ctrl, (int)sh.scan_total);
        }
        __syncthreads();
        const uint32_t m1 = tid < nwords ? (uint32_t)__popc(hmarks[tid]) : 0u;
        const uint32_t p1 = block_scan_excl(m1, sh.scan, &sh.scan_total);
        if (tid < nwords) hwpfx[tid] = p1;
        if (tid == 0) sh.n_hpatch = (int)sh.scan_total;
        __syncthreads();
    }
    // ---- scatter the beams into their buckets; count the hits of every hit patch -------------------------------------
    for (int b = tid; b < n; b += blockDim.x) {
        const uint64_t key = keys[b];
        if (key != ~0ull) {
            uint32_t sb = (uint32_t)((key >> 16) >> 31) & 0x1FFu;
            sb = sb > 255u ? 255u : sb;
            sorted[atomicAdd(&bfill[pull_key_class(key) * 256 + (int)sb], 1u)] = key;
        }
        const uint32_t hr = hrec[b];
        if (hr != ~0u) {
            const uint32_t di = hr >> 10;
            const uint32_t ho = hwpfx[di >> 5] + (uint32_t)__popc(hmarks[di >> 5] & ((1u << (di & 31)) - 1u));
            atomicAdd(&hcnt[ho], 1u);
        }
    }
    __syncthreads();
    const int n_list = sh.n_list;
    // ---- exact order: odd-even transposition until a full round changes nothing ------------------------------------
    for (;;) {
        if (tid == 0) sh.swapped = 0;
        __syncthreads();
        bool sw = false;
        for (int i = 2 * tid; i + 1 < n_list; i += 2 * blockDim.x) {
            const uint64_t x = sorted[i], y = sorted[i + 1];
            if (x > y) { sorted[i] = y; sorted[i + 1] = x; sw = true; }
        }
        __syncthreads();
        for (int i = 2 * tid + 1; i + 1 < n_list; i += 2 * blockDim.x) {
            const uint64_t x = sorted[i], y = sorted[i + 1];
            if (x > y) { sorted[i] = y; sorted[i + 1] = x; sw = true; }
        }
        if (sw) sh.swapped = 1;
        __syncthreads();
        const bool again = sh.swapped != 0;
        __syncthreads();
        if (!again) break;
    }
    // ---- class lists to global memory ------------------------------------------------------------------------------------
    PullEntry* glist = pv.list + (size_t)blockIdx.x * pv.stride;
    uint32_t* ghits  = pv.hits + (size_t)blockIdx.x * pv.stride;
    for (int i = tid; i < n_list; i += blockDim.x) {
        const uint64_t k = sorted[i];
        const uint32_t beam = pull_key_beam(k);
        glist[i] = PullEntry{ndb[beam], beam, pull_magic(ndb[beam] & 0xFFFFu)};
        const int cls = pull_key_class(k), prev = i ? pull_key_class(sorted[i - 1]) : -1;
        for (int c = prev + 1; c <= cls; ++c) sh.prefix[c] = i;
        if (i == n_list - 1)
            for (int c = cls + 1; c <= 8; ++c) sh.prefix[c] = n_list;
    }
    // ---- hit records grouped by hit patch ---------------------------------------------------------------------------------
    {
        const int nhp = sh.n_hpatch, per = (nhp + (int)blockDim.x - 1) / (int)blockDim.x;
        uint32_t sum = 0;
        for (int k = 0; k < per; ++k) {
            const int i = tid * per + k;
            if (i < nhp) sum += hcnt[i];
        }
        uint32_t base = block_scan_excl(sum, sh.scan, &sh.scan_total);
        for (int k = 0; k < per; ++k) {
            const int i = tid * per + k;
            if (i < nhp) { const uint32_t c = hcnt[i]; hcnt[i] = base; base += c; }
        }
        if (tid == 0) {
            sh.n_hits = (int)sh.scan_total;
            hcnt[nhp] = sh.scan_total;
        }
        __syncthreads();
    }
    for (int b = tid; b < n; b += blockDim.x) {
        const uint32_t hr = hrec[b];
        if (hr == ~0u) continue;
        const uint32_t di = hr >> 10;
        const uint32_t ho = hwpfx[di >> 5] + (uint32_t)__popc(hmarks[di >> 5] & ((1u << (di & 31)) - 1u));
        ghits[hcnt[ho] + atomicAdd(&hfill[ho], 1u)] = pull_hit_record(hr & (kPatchCells - 1), (uint32_t)b);
    }
    // ---- one task per marked patch (the tasks of a particle stay together) ---------------------------------------------------
    for (int w = tid; w < nwords; w += blockDim.x) {
        uint32_t bits = marks[w];
        uint32_t k = (uint32_t)sh.task_base + wpfx[w];
        while (bits) {
            const int bit = __ffs(bits) - 1;
            bits &= bits - 1;
            const uint32_t di = (uint32_t)(w * 32 + bit);
            uint32_t hw = 0;
            if ((hmarks[w] >> bit) & 1u) {
                const uint32_t ho = hwpfx[w] + (uint32_t)__popc(hmarks[w] & ((1u << bit) - 1u));
                hw = (hcnt[ho] << 16) | (hcnt[ho + 1] - hcnt[ho]);
            }
            pv.tasks[k++] = make_uint2(((uint32_t)blockIdx.x << 16) | di, hw);
        }
    }
    __syncthreads();
    if (tid == 0) {
        hdr->ox = (int32_t)ox;
        hdr->oy = (int32_t)oy;
        for (int c = 0; c < 9; ++c) hdr->prefix[c] = sh.prefix[c];
        hdr->n_hits    = sh.n_hits;
        hdr->ok        = 1;
        hdr->task_base = sh.task_base;
        hdr->n_tasks   = sh.n_tasks;
        MapUpdateStats& st = stats[blockIdx.x];
        st.ray_cells   = sh.cells;
        st.log_records = 0;
        st.events      = 0;   // k_ray_pull appends the obstacle events of this particle and counts them here
        st.dm_pops     = 0;
    }
}

// k_ray_pull: persistent CTAs take work units (particle, every splits-th patch of it), stage the particle's class lists and hit
// records in shared memory with TMA bulk copies, and their warps then take patches one by one.  Per patch: the axis passes fill
// the count tile, plain cells get `visited += count` (log-odds maps: `count` misses) with row-coalesced read-modify-writes of the
// patch the particle owns exclusively, candidate cells (hit in this scan, or distance-map obstacles) are compacted and replayed in
// beam order, one lane per cell.  A patch without any touched cell is neither allocated nor detached (the reference would not have
// created it).
constexpr int kPullWarps = 8;
constexpr int kPullCandCap = 512;
constexpr int kTileStride = kPatchLen + 2;   // uint16 counters, rows 34 apart: column-wise and row-wise accesses are both conflict free
struct PullWarpShared {
    uint16_t tile[kPatchLen * kTileStride];   // crossing count of cell (r, c) at [r * 34 + c]
    uint32_t hitbits[kPatchLen];              // cells of the patch that are hit cells of this scan
    uint16_t cand[kPullCandCap];              // compacted candidate cells
};
struct PullCtaShared {
    RayPullHeader hdr;
    uint64_t bar;
    int unit, next;
};
struct RayPullLayout {
    size_t list, hits, warps, total;
    __host__ __device__ explicit RayPullLayout(int n_beams)
    {
        const size_t cap = ((size_t)n_beams + 31) & ~(size_t)31;
        size_t o = (sizeof(PullCtaShared) + 15) & ~(size_t)15;
        list = o;  o += cap * sizeof(PullEntry);
        hits = o;  o += cap * 4;
        warps = o; o += (size_t)kPullWarps * sizeof(PullWarpShared);
        total = o;
    }
};

// Ordered replay of the compacted candidate cells of one patch, one lane per cell (kept out of line: it is the rare path and
// would otherwise be inlined twice into k_ray_pull, whose hot loops then fall out of the instruction cache).  Returns true when a
// cell became a distance-map obstacle.
template <bool kProb>
static __device__ __noinline__ bool pull_replay_patch(const StoreView& s, const RayParams& rp, const PullEntry* list, const int* prefix, const uint32_t* hits, int h_lo, int h_hi,
                                                      const uint16_t* cand, int ncand, uint32_t* patch, int slot, int cx0, int cy0, int px, int py,
                                                      MapUpdateStats* st, uint64_t* events, int lane)
{
    bool newhot = false;
    for (int k = lane; k < ncand; k += 32) {
        const uint32_t ci = cand[k];
        const int r = (int)(ci >> kPatchLog2), c = (int)(ci & (kPatchLen - 1));
        const PullRuns runs = pull_cell_runs(list, prefix, cx0 + c, cy0 + r);
        uint32_t* fword = fbits_ptr(s, slot) + r;
        const bool before = (__ldcg(fword) >> c) & 1u;
        bool obstacle = before;
        const uint32_t key = ((uint32_t)(py * kPatchLen + r) << 16) | (uint32_t)(px * kPatchLen + c);   // window-relative cell
        auto emit = [&](bool add, uint32_t seq) {
            const uint32_t idx = atomicAdd(&st->events, 1u);
            if (idx < (uint32_t)rp.event_cap) events[idx] = push_record((seq << 1) | (add ? 1u : 0u), key);
        };
        uint32_t* cell = patch + ci;
        if (!kProb) {
            *cell = pull_replay_cell(list, runs, hits, h_lo, h_hi, ci, *cell, obstacle, emit);
        } else {
            *cell = __float_as_uint(pull_replay_cell_prob(list, runs, hits, h_lo, h_hi, ci, __uint_as_float(*cell), obstacle, rp.prob, emit));
            atomicOr(kbits_ptr(s, slot) + r, 1u << c);
        }
        if (obstacle != before) {
            if (obstacle) {
                atomicOr(fword, 1u << c);
                newhot = true;
            } else {
                atomicAnd(fword, ~(1u << c));
            }
        }
    }
    __syncwarp();
    return newhot;
}

#ifndef LAMA_PULL_MIN_CTAS
#define LAMA_PULL_MIN_CTAS 4
#endif
constexpr int kPullCtasPerSm = LAMA_PULL_MIN_CTAS;   // resident CTAs per SM the register budget is sized for (4: 64 registers, 2: 128)
template <bool kProb>
__global__ void __launch_bounds__(kPullWarps * 32, kPullCtasPerSm)
k_ray_pull(StoreView s, RayParams rp, int count, uint64_t* __restrict__ events_out, MapUpdateStats* __restrict__ stats)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const RayPullView& pv = rp.pull;
    const RayPullLayout L(rp.scan.n_beams);
    PullCtaShared& sh   = *reinterpret_cast<PullCtaShared*>(smem_raw);
    PullEntry* list     = reinterpret_cast<PullEntry*>(smem_raw + L.list);
    uint32_t* hits      = reinterpret_cast<uint32_t*>(smem_raw + L.hits);
    PullWarpShared& w   = reinterpret_cast<PullWarpShared*>(smem_raw + L.warps)[warp];
    const RayPullHeader* hdr = &sh.hdr;
    const int dim = s.window.dim, S = pv.splits;
    int log2dim = 0;
    while ((1 << (log2dim + 1)) <= dim) ++log2dim;
    if (tid == 0) mbar_init(&sh.bar, 1);
    uint32_t err = 0, parity = 0;
    for (;;) {
        __syncthreads();   // every warp is done with the staged data of the previous unit
        if (tid == 0) sh.unit = atomicAdd(pv.ctrl + 1, 1);
        __syncthreads();
        const int unit = sh.unit;
        if (unit >= count * S) break;
        const int pl = unit / S, split = unit - pl * S;
        if (!__ldcg(&pv.hdr[pl].ok)) continue;   // k_raycast handles this particle
        if (tid == 0) {
            sh.hdr  = pv.hdr[pl];
            sh.next = 0;
            const uint32_t b0 = (uint32_t)sh.hdr.prefix[8] * (uint32_t)sizeof(PullEntry), b1 = ((uint32_t)sh.hdr.n_hits * 4u + 15u) & ~15u;
            mbar_expect_tx(&sh.bar, b0 + b1);
            if (b0) tma_load_1d(list, pv.list + (size_t)pl * pv.stride, b0, &sh.bar);
            if (b1) tma_load_1d(hits, pv.hits + (size_t)pl * pv.stride, b1, &sh.bar);
        }
        mbar_wait(&sh.bar, parity);
        parity ^= 1u;
        __syncthreads();   // sh.hdr / sh.next written by thread 0
        const int n_tasks = hdr->n_tasks, ox = hdr->ox, oy = hdr->oy;
        int32_t* gdir = dir_of(s, rp.set, rp.particle_offset + pl, kMapOcc);
        for (;;) {
            int t = 0;
            if (lane == 0) t = atomicAdd(&sh.next, 1);
            t = __shfl_sync(0xffffffffu, t, 0);
            const int ti = split + t * S;
            if (ti >= n_tasks) break;
            const uint2 task = __ldg(pv.tasks + hdr->task_base + ti);
            const int di = (int)(task.x & 0xFFFFu), h_lo = (int)(task.y >> 16), h_hi = h_lo + (int)(task.y & 0xFFFFu);
            const int px = di & (dim - 1), py = di >> log2dim;
            const int cx0 = px * kPatchLen - ox, cy0 = py * kPatchLen - oy;
            {   // zero the count tile (2 176 bytes)
                uint32_t* tz = reinterpret_cast<uint32_t*>(w.tile);
#pragma unroll
                for (int i = 0; i < kPatchLen * kTileStride / 2 / 32; ++i) tz[i * 32 + lane] = 0u;
            }
            w.hitbits[lane] = 0u;
            __syncwarp();
            bool touched = false;
            {   // x-major classes: lane = column.  All lanes run over the same beams; each beam lands in one row of the lane's column.
                const int m = cx0 + lane;
                const uint32_t a = (uint32_t)(m < 0 ? -m : m);
                pull_patch_classes(list, hdr->prefix, 0, cx0, cy0, [&](int, bool mneg, bool tneg, int lo, int hi) {
                    if (m == 0 || (m < 0) != mneg) return;
                    for (int i = lo; i < hi; ++i) {
                        const int pos = pull_land(list[i], a, tneg, cy0);
                        if (pos >= 0) {
                            ++w.tile[pos * kTileStride + lane];
                            touched = true;
                        }
                    }
                });
            }
            __syncwarp();
            {   // y-major classes: lane = row
                const int m = cy0 + lane;
                const uint32_t a = (uint32_t)(m < 0 ? -m : m);
                pull_patch_classes(list, hdr->prefix, 4, cy0, cx0, [&](int, bool mneg, bool tneg, int lo, int hi) {
                    if (m == 0 || (m < 0) != mneg) return;
                    for (int i = lo; i < hi; ++i) {
                        const int pos = pull_land(list[i], a, tneg, cx0);
                        if (pos >= 0) {
                            ++w.tile[lane * kTileStride + pos];
                            touched = true;
                        }
                    }
                });
            }
            for (int i = h_lo + lane; i < h_hi; i += 32) {
                const uint32_t cell = pull_hit_cell(hits[i]);
                atomicOr(&w.hitbits[cell >> 5], 1u << (cell & 31));
            }
            __syncwarp();
            if (!__any_sync(0xffffffffu, touched) && h_hi == h_lo) continue;   // nothing of this scan lands in the patch

            // Map::get (mutable): allocate on first touch, detach a shared patch (map.cpp:400-408, cow_ptr.h:104-114)
            const int e0 = gdir[di];
            const bool hot = e0 >= 0 && (e0 & kDirHot);
            const int slot = warp_make_exclusive(s, gdir, gdir, di, lane);
            if (slot < 0) {
                err |= kErrPoolEmpty;
                continue;
            }
            uint32_t* patch = patch_ptr(s, slot);
            const uint32_t hitrow  = w.hitbits[lane];                                            // lane = row
            const uint32_t candrow = hitrow | (hot ? __ldcg(fbits_ptr(s, slot) + lane) : 0u);   // | cells that are distance-map obstacles
            int ncand = 0;
            bool newhot = false;
            auto replay_candidates = [&]() {
                newhot |= pull_replay_patch<kProb>(s, rp, list, hdr->prefix, hits, h_lo, h_hi, w.cand, ncand, patch, slot, cx0, cy0, px, py, stats + pl,
                                                   events_out + (size_t)pl * rp.event_cap, lane);
                ncand = 0;
            };
            for (int r0 = 0; r0 < kPatchLen; r0 += 8) {
                uint32_t v[8];   // eight rows of the patch in flight at once
#pragma unroll
                for (int k = 0; k < 8; ++k) v[k] = __ldcg(patch + (r0 + k) * kPatchLen + lane);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const int r = r0 + k;
                    const uint32_t cnt = w.tile[r * kTileStride + lane];
                    const uint32_t cw = __shfl_sync(0xffffffffu, candrow, r);
                    bool plain = cnt != 0u;   // misses only, never an obstacle: counter additions commute
                    if (cw != 0u) {           // (rare) the row holds candidate cells
                        const uint32_t hw = __shfl_sync(0xffffffffu, hitrow, r);
                        const bool iscand = (cw >> lane) & 1u, touch = cnt != 0u || ((hw >> lane) & 1u);
                        plain = touch && !iscand;
                        const uint32_t m = __ballot_sync(0xffffffffu, touch && iscand);
                        if (m) {
                            if (ncand + 32 > kPullCandCap) replay_candidates();
                            if (touch && iscand) w.cand[ncand + __popc(m & ((1u << lane) - 1u))] = (uint16_t)(r * kPatchLen + lane);
                            ncand += __popc(m);
                        }
                    }
                    if (plain) {
                        uint32_t* cell = patch + r * kPatchLen + lane;
                        if (!kProb) {
                            *cell = v[k] + (cnt << 16);   // visited += cnt (wraps like the reference's uint16)
                        } else {
                            float p = __uint_as_float(v[k]);
                            for (uint32_t q = cnt; q > 0; --q) p = prob_miss(p, rp.prob);
                            *cell = __float_as_uint(p);
                        }
                    }
                    if (kProb) {
                        const uint32_t known = __ballot_sync(0xffffffffu, plain);
                        if (lane == 0 && known) kbits_ptr(s, slot)[r] |= known;
                    }
                }
            }
            __syncwarp();
            if (ncand) replay_candidates();
            if (__any_sync(0xffffffffu, newhot) && !hot && lane == 0) gdir[di] |= kDirHot;   // from now on the patch may hold obstacle bits
            __syncwarp();
        }
    }
    err = __reduce_or_sync(0xffffffffu, err);
    if (lane == 0 && err) atomicOr(s.status, err);
}

constexpr int kBrushThreads = 128;   // four warps sort the events and warm the L1; then warp 0 alone runs the sequential brushfire
__global__ void __launch_bounds__(kBrushThreads)
k_brushfire(StoreView s, BrushParams bp, const uint64_t* __restrict__ events, MapUpdateStats* __restrict__ stats)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int dim2    = s.window.dim * s.window.dim;
    int32_t* dir      = reinterpret_cast<int32_t*>(smem_raw);
    uint64_t* lower_h = reinterpret_cast<uint64_t*>(smem_raw + (size_t)dim2 * 4);   // 16-byte aligned: dim2 * 4 is a multiple of 16
    uint64_t* raise_h = lower_h + bp.lower_cap + 2;
    uint64_t* ev      = raise_h + bp.raise_cap + 2;                                 // the events of this particle, sorted here
    uint32_t* scratch = reinterpret_cast<uint32_t*>(ev + bp.event_cap);
    uint64_t* bar     = reinterpret_cast<uint64_t*>(scratch + 32);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const int particle = bp.particle_offset + blockIdx.x;
    int32_t* gdir      = dir_of(s, bp.set, particle, kMapDm);

#ifdef LAMA_PHASE_TIMING
    long long bt[5] = {clock64(), 0, 0, 0, 0};
#endif
    if (tid == 0) mbar_init(bar, 1);
    __syncthreads();
    // The obstacle events arrive in any order (k_ray_pull appends them cell by cell): sorting by their (beam, step) stamp restores
    // the reference's addObstacle / removeObstacle call sequence (ray_core.h).
    uint32_t nev = stats[blockIdx.x].events;
    uint32_t my_err = 0;
    if (nev > (uint32_t)bp.event_cap) {
        my_err |= kErrPushOverflow;
        nev = (uint32_t)bp.event_cap;
    }
    const uint64_t* gev = events + (size_t)blockIdx.x * bp.event_cap;
    const int evpad = next_pow2((int)nev);
    for (int i = tid; i < evpad; i += blockDim.x) ev[i] = i < (int)nev ? gev[i] : ~0ull;
    __syncthreads();
    block_bitonic_sort(ev, evpad);
    block_stage_tma(dir, gdir, (uint32_t)dim2 * 4u, bar, 0);

    // The L1 is cold at every launch and the waves started by the events stay within `reach` cells of them: pull the patch of
    // every event (32 rows = 32 lines, one per lane) and the neighbouring patches a wave can reach into L1 before the sequential
    // part starts, so that its dependent loads hit (ncu: 24 % of the loads missed L1, 21 % of the stall samples waited for them).
    {
        int reach = 0;
        while ((uint32_t)(reach * reach) < bp.max_sqdist) ++reach;
        const int dim = s.window.dim;
        for (uint32_t i = warp; i < nev; i += nwarps) {
            const uint32_t key = (uint32_t)ev[i];
            const int x = (int)(key & 0xFFFFu), y = (int)(key >> 16);
            const int px = x >> kPatchLog2, py = y >> kPatchLog2, cx = x & (kPatchLen - 1), cy = y & (kPatchLen - 1);
            const int x0 = cx < reach ? -1 : 0, x1 = cx >= kPatchLen - reach ? 1 : 0, y0 = cy < reach ? -1 : 0, y1 = cy >= kPatchLen - reach ? 1 : 0;
            for (int dy = y0; dy <= y1; ++dy)
                for (int dx = x0; dx <= x1; ++dx) {
                    const int qx = px + dx, qy = py + dy;
                    if ((unsigned)qx >= (unsigned)dim || (unsigned)qy >= (unsigned)dim) continue;
                    const int e = dir[qy * dim + qx];
                    if (e < 0) continue;
                    const uint32_t* row = patch_ptr(s, e & kDirSlotMask) + lane * kPatchLen;
                    asm volatile("prefetch.global.L1 [%0];" ::"l"(row));
                }
        }
    }
    if (warp != 0) return;
#ifdef LAMA_PHASE_TIMING
    bt[1] = clock64();
#endif

    WarpBrushfire bf(s, dir, gdir, scratch, lane, SmemHeap{lower_h, 0u, (uint32_t)bp.lower_cap}, SmemHeap{raise_h, 0u, (uint32_t)bp.raise_cap},
                     bp.max_sqdist);
    bf.err |= my_err;
    for (uint32_t i = 0; i < nev; ++i) {
        const uint64_t e   = ev[i];
        const uint32_t key = (uint32_t)e;  // window-relative cell
        if ((e >> 32) & 1u) bf.add_obstacle(key & 0xFFFFu, key >> 16);
        else bf.remove_obstacle(key & 0xFFFFu, key >> 16);
    }
#ifdef LAMA_PHASE_TIMING
    bt[2] = clock64();
    const uint32_t q0 = bf.raise_q.size, q1 = bf.lower_q.size;
#endif
    const uint32_t processed = bf.update();
#ifdef LAMA_PHASE_TIMING
    bt[3] = clock64();
    if (lane == 0 && bp.debug) printf("bf %d: pre %lld events %lld update %lld | nev %u raise %u lower %u pops %u\n", blockIdx.x, bt[1] - bt[0], bt[2] - bt[1], bt[3] - bt[2], nev, q0, q1, processed);
    if (lane == 0 && bp.debug) printf("bfc %d: pop %lld cur %lld nbr %lld chk %lld commit %lld (pushes %lld)\n", blockIdx.x, bf.cyc[0], bf.cyc[1], bf.cyc[2], bf.cyc[3], bf.cyc[4], bf.cyc[5]);
#endif
    const uint32_t err = __reduce_or_sync(0xffffffffu, bf.err);
    if (lane == 0) {
        stats[blockIdx.x].dm_pops = processed;
        if (err) atomicOr(s.status, err);
    }
}

// ==================================================================================================
// resampling / bookkeeping kernels
// ==================================================================================================
__global__ void k_copy_dirs(StoreView s, int src_set, int dst_set, const int32_t* __restrict__ idx, int dst_first)
{
    const int p = dst_first + blockIdx.x, kind = blockIdx.y;
    const int dim2 = s.window.dim * s.window.dim;
    const int a  = idx[blockIdx.x];
    int32_t* src = dir_of(s, src_set, a < 0 ? 0 : a, kind);
    int32_t* dst = dir_of(s, dst_set, p, kind);
    for (int e = threadIdx.x; e < dim2; e += blockDim.x) {
        int slot = a < 0 ? -1 : src[e];
        if (slot >= 0) {
            atomicAdd(&s.refcount[slot & kDirSlotMask], 1);
            // shared from now on: neither copy owns it (several blocks may clear the same source entry: same value)
            if ((slot & kDirOwn) && src_set == dst_set) src[e] = slot & ~kDirOwn;
            slot &= ~kDirOwn;  // keeps kDirHot
        }
        dst[e] = slot;
    }
}
__global__ void k_release(StoreView s, int set, int first)
{
    const int p = first + blockIdx.x, kind = blockIdx.y;
    const int dim2 = s.window.dim * s.window.dim;
    int32_t* d = dir_of(s, set, p, kind);
    for (int e = threadIdx.x; e < dim2; e += blockDim.x) {
        int slot = d[e];
        if (slot >= 0) {
            release_slot(s, slot & kDirSlotMask);
            d[e] = -1;
        }
    }
}
// Map::deletePatchAt (map.cpp:465-488) for a list of directory entries, in every map kind of one particle
__global__ void k_delete_patches(StoreView s, int set, int particle, const int32_t* __restrict__ list)
{
    const int di = list[blockIdx.x];
    if (threadIdx.x != 0) return;
    for (int kind = 0; kind < s.n_kinds; ++kind) {
        int32_t* d = dir_of(s, set, particle, kind);
        const int e = d[di];
        if (e >= 0) {
            release_slot(s, e & kDirSlotMask);
            d[di] = -1;
        }
    }
}

// the per-particle payload of the sharded exchange: {state (4), likelihood, reference evaluations, iterations}, then one digest word
__global__ void k_pack_results(const MatchResult* __restrict__ res, int n, double digest, double* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const MatchResult& r = res[i];
        double* o = out + (size_t)i * kShardFields;
        o[0] = r.state.c; o[1] = r.state.s; o[2] = r.state.tx; o[3] = r.state.ty;
        o[4] = r.sums[11];
        o[5] = (double)r.evals_ref;
        o[6] = (double)r.iterations;
    }
    if (i == 0) out[(size_t)n * kShardFields] = digest;
}

__global__ void k_merge_free(StoreView s)
{
    __shared__ int n, base;
    if (threadIdx.x == 0) {
        n    = *s.freed_count;
        base = *s.free_count;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) s.free_slots[base + i] = s.freed[i];
    __syncthreads();
    if (threadIdx.x == 0) {
        *s.free_count  = base + n;
        *s.freed_count = 0;
        s.ray_ctrl[0] = s.ray_ctrl[1] = 0;   // task list of the pull ray cast: empty for the next scan
    }
}
__global__ void k_init_store(StoreView s, int n_sets)
{
    const size_t total_dir = (size_t)n_sets * s.n_particles * s.n_kinds * s.window.dim * s.window.dim;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total_dir; i += (size_t)gridDim.x * blockDim.x) s.dirs[i] = -1;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)s.n_slots; i += (size_t)gridDim.x * blockDim.x) {
        s.free_slots[i] = s.n_slots - 1 - (int)i;  // slot 0 is handed out first
        s.refcount[i]   = 0;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        *s.free_count  = s.n_slots;
        *s.freed_count = 0;
        *s.status      = 0;
        s.counters[0] = s.counters[1] = s.counters[2] = 0;
    }
}

__global__ void k_export(StoreView s, int set, int particle, int kind, uint32_t x0, uint32_t y0, int w, int h, uint32_t* __restrict__ out,
                         uint8_t* __restrict__ present)
{
    const int32_t* d = dir_of(s, set, particle, kind);
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < w * h; k += gridDim.x * blockDim.x) {
        uint32_t x = x0 + (uint32_t)(k % w), y = y0 + (uint32_t)(k / w);
        int di   = dir_index(s.window, x, y);
        int slot = di < 0 ? -1 : d[di];
        out[k]   = slot < 0 ? 0u : __ldcg(patch_ptr(s, slot & kDirSlotMask) + cell_index(x, y));
        if (present) present[k] = slot >= 0;
    }
}

// the words of n scattered cells of one map; flags bit 0: the patch exists, bit 1: the cell's bit in the `known` plane (log-odds maps)
__global__ void k_gather_cells(StoreView s, int set, int particle, int kind, const uint32_t* __restrict__ cells, int n, uint32_t* __restrict__ words,
                               uint8_t* __restrict__ flags)
{
    const int32_t* d = dir_of(s, set, particle, kind);
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const uint32_t x = cells[2 * k], y = cells[2 * k + 1];
        const int di   = dir_index(s.window, x, y);
        const int slot = di < 0 ? -1 : d[di];
        uint32_t w = 0;
        uint8_t f = 0;
        if (slot >= 0) {
            const uint32_t ci = cell_index(x, y);
            w = __ldcg(patch_ptr(s, slot & kDirSlotMask) + ci);
            f = 1;
            if (kind == kMapOcc && s.kbits && ((__ldcg(kbits_ptr(s, slot & kDirSlotMask) + (ci >> 5)) >> (ci & 31)) & 1u)) f |= 2;
        }
        words[k] = w;
        flags[k] = f;
    }
}

__global__ void k_export_bits(StoreView s, int plane, int set, int particle, uint32_t x0, uint32_t y0, int w, int h, uint8_t* __restrict__ out)
{
    const int32_t* d = dir_of(s, set, particle, kMapOcc);
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < w * h; k += gridDim.x * blockDim.x) {
        uint32_t x = x0 + (uint32_t)(k % w), y = y0 + (uint32_t)(k / w);
        int di   = dir_index(s.window, x, y);
        int slot = di < 0 ? -1 : d[di];
        uint8_t v = 0;
        const uint32_t* base = plane == 0 ? s.fbits : s.kbits;
        if (slot >= 0 && base) {
            const uint32_t ci = cell_index(x, y);
            v = (__ldcg(base + (size_t)(slot & kDirSlotMask) * 32 + (ci >> 5)) >> (ci & 31)) & 1u;
        }
        out[k] = v;
    }
}

// one warp per patch of the (patch-aligned) window
__global__ void k_import(StoreView s, int set, int particle, int kind, uint32_t x0, uint32_t y0, int w, int h, const uint32_t* __restrict__ in)
{
    const int lane = threadIdx.x & 31;
    const int pw = w / kPatchLen, ph = h / kPatchLen;
    const int pi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (pi >= pw * ph) return;
    const int px = pi % pw, py = pi / pw;
    int32_t* d = dir_of(s, set, particle, kind);
    // does the patch hold anything?
    uint32_t any = 0;
    for (int c = lane; c < kPatchCells; c += 32) {
        int cx = c & (kPatchLen - 1), cy = c >> kPatchLog2;
        any |= in[(size_t)(py * kPatchLen + cy) * w + px * kPatchLen + cx];
    }
    any = __reduce_or_sync(0xffffffffu, any);
    if (!any) return;
    const uint32_t x = x0 + px * kPatchLen, y = y0 + py * kPatchLen;
    int di = dir_index(s.window, x, y);
    if (di < 0) {
        if (lane == 0) atomicOr(s.status, kErrWindow);
        return;
    }
    int slot = warp_make_exclusive(s, d, d, di, lane);
    if (slot < 0) return;
    uint32_t* dst = patch_ptr(s, slot);
    for (int c = lane; c < kPatchCells; c += 32) {
        int cx = c & (kPatchLen - 1), cy = c >> kPatchLog2;
        dst[c] = in[(size_t)(py * kPatchLen + cy) * w + px * kPatchLen + cx];
    }
}

// gather the patches listed in `slots` into a contiguous buffer (particle migration between GPUs, checkpoints); out_kbits (may be null)
// also takes the known plane of a store that has one
__global__ void k_gather_patches(StoreView s, const int32_t* __restrict__ slots, int n, uint32_t* __restrict__ out, uint32_t* __restrict__ out_fbits,
                                 uint32_t* __restrict__ out_kbits)
{
    const int lane = threadIdx.x & 31;
    const int pi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (pi >= n) return;
    const int slot = slots[pi] & kDirSlotMask;
    warp_copy_patch(out + (size_t)pi * kPatchCells, patch_ptr(s, slot), lane);
    out_fbits[(size_t)pi * 32 + lane] = __ldcg(fbits_ptr(s, slot) + lane);
    if (out_kbits && s.kbits) out_kbits[(size_t)pi * 32 + lane] = __ldcg(kbits_ptr(s, slot) + lane);
}

// ---- checkpoint: count the references of every slot, compact the slots in use, rewrite the directories ---------------------------------
// one thread per directory entry of `set` (every particle, every kind incl. the log-odds scratch kind): cnt[slot] += 1 per reference.
// bad bit 0: an entry whose slot lies outside the pool
__global__ void k_ckpt_count(StoreView s, int set, int32_t* __restrict__ cnt, uint32_t* __restrict__ bad)
{
    const size_t n = (size_t)s.n_particles * s.n_kinds * s.window.dim * s.window.dim;
    const int32_t* d = dir_of(s, set, 0, 0);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int32_t e = d[i];
        if (e < 0) continue;
        const int32_t slot = e & kDirSlotMask;
        if (slot >= s.n_slots) { atomicOr(bad, 1u); continue; }
        atomicAdd(&cnt[slot], 1);
    }
}
// one thread per slot: used[slot] = 1 when a directory references it.  bad bit 1: the count differs from the slot's reference count
// (a store that is not self-consistent is never written)
__global__ void k_ckpt_mark(StoreView s, const int32_t* __restrict__ cnt, int32_t* __restrict__ used, uint32_t* __restrict__ bad)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < s.n_slots; i += gridDim.x * blockDim.x) {
        const int32_t c = cnt[i];
        used[i] = c > 0 ? 1 : 0;
        if (c != s.refcount[i]) atomicOr(bad, 2u);
    }
}
// after the exclusive scan (new_id = number of used slots below): list[new_id] = old slot, ref[new_id] = its reference count
__global__ void k_ckpt_list(StoreView s, const int32_t* __restrict__ used, const int32_t* __restrict__ new_id, int32_t* __restrict__ list,
                            int32_t* __restrict__ ref)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < s.n_slots; i += gridDim.x * blockDim.x)
        if (used[i]) {
            list[new_id[i]] = i;
            ref[new_id[i]]  = s.refcount[i];
        }
}
// one thread per directory entry of `set`: out = new id | the entry's flags (kDirHot and kDirOwn kept exactly); the store is not written
__global__ void k_ckpt_remap(StoreView s, int set, const int32_t* __restrict__ new_id, int32_t* __restrict__ out)
{
    const size_t n = (size_t)s.n_particles * s.n_kinds * s.window.dim * s.window.dim;
    const int32_t* d = dir_of(s, set, 0, 0);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int32_t e = d[i];
        out[i] = e < 0 ? -1 : (new_id[e & kDirSlotMask] | (e & ~kDirSlotMask));
    }
}
// allocate a patch per listed directory entry of (set, particle, kind) and fill it from `in`
__global__ void k_scatter_patches(StoreView s, int set, int particle, int kind, const int32_t* __restrict__ entries, int n, const uint32_t* __restrict__ in,
                                  const uint32_t* __restrict__ in_fbits)
{
    const int lane = threadIdx.x & 31;
    const int pi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (pi >= n) return;
    int32_t* d = dir_of(s, set, particle, kind);
    int slot = warp_make_exclusive(s, d, d, entries[pi], lane);
    if (slot < 0) return;
    warp_copy_patch(patch_ptr(s, slot), in + (size_t)pi * kPatchCells, lane);
    const uint32_t fb = in_fbits[(size_t)pi * 32 + lane];
    fbits_ptr(s, slot)[lane] = fb;
    if (kind == kMapOcc && __any_sync(0xffffffffu, fb != 0u) && lane == 0) d[entries[pi]] |= kDirHot;
}

// Loc2D::addSamplingCovariance (src/loc2d.cpp:199-236): for every sampling offset the likelihood
//   l = sum over every `stride`-th beam of exp(-d^2 / 0.01)^3,  d = nearest-cell distance at the offset pose.
// One block per offset; the host accumulates K, u, s in the reference's order.
__global__ void k_sampling(StoreView s, int set, int particle, const double* __restrict__ points, ScanParams scan, SE2 pose, const double* __restrict__ offsets,
                           int stride, double resolution, uint32_t max_sqdist, double* __restrict__ out)
{
    __shared__ Affine tf;
    __shared__ double part[8];
    const int32_t* d = dir_of(s, set, particle, kMapDm);
    if (threadIdx.x == 0) {
        SE2 st = pose;
        st.tx = add_rn(pose.tx, offsets[2 * blockIdx.x]);
        st.ty = add_rn(pose.ty, offsets[2 * blockIdx.x + 1]);
        tf = compose_tf(st, scan.moving);
    }
    __syncthreads();
    const double dmax = mul_rn(sqrt((double)max_sqdist), resolution);
    double l = 0.0;
    for (int k = threadIdx.x * stride; k < scan.n_beams; k += blockDim.x * stride) {
        double hit[3];
        apply_tf(tf, points[3 * k], points[3 * k + 1], points[3 * k + 2], hit);
        const uint32_t x = w2m(hit[0], scan.scale), y = w2m(hit[1], scan.scale);
        const int di = dir_index(s.window, x, y);
        const int slot = di < 0 ? -1 : d[di];
        const uint32_t w = slot < 0 ? 0u : __ldcg(patch_ptr(s, slot & kDirSlotMask) + cell_index(x, y));
        const double dist = (w & kDmValid) ? mul_rn(sqrt((double)dm_sqdist(w)), resolution) : dmax;
        const double e = exp(-mul_rn(dist, dist) / 0.01);
        l += e * e * e;
    }
    l = warp_sum(l);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = l;
    __syncthreads();
    if (threadIdx.x == 0) {
        double v = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += part[w];
        out[blockIdx.x] = v;
    }
}

// MatchSurface2D::error() (src/match_surface_2d.cpp:92-116): sqrt(sum d^2 / N) with d the NEAREST-cell distance (w2m rounding +
// DynamicDistanceMap::distance(Vector3ui), dynamic_distance_map.cpp:140-147) of every point at the given state.  One block per state.
__global__ void k_match_error(StoreView s, int set, int particle0, int shared_map, const double* __restrict__ points, ScanParams scan, const SE2* __restrict__ states,
                              double resolution, uint32_t max_sqdist, double* __restrict__ out)
{
    __shared__ Affine tf;
    __shared__ double part[8];
    const int32_t* d = dir_of(s, set, shared_map ? particle0 : particle0 + blockIdx.x, kMapDm);
    if (threadIdx.x == 0) tf = compose_tf(states[blockIdx.x], scan.moving);
    __syncthreads();
    const double dmax = mul_rn(sqrt((double)max_sqdist), resolution);
    double acc = 0.0;
    for (int k = threadIdx.x; k < scan.n_beams; k += blockDim.x) {
        double hit[3];
        apply_tf(tf, points[3 * k], points[3 * k + 1], points[3 * k + 2], hit);
        const uint32_t x = w2m(hit[0], scan.scale), y = w2m(hit[1], scan.scale);
        const int di = dir_index(s.window, x, y);
        const int slot = di < 0 ? -1 : d[di];
        const uint32_t w = slot < 0 ? 0u : __ldcg(patch_ptr(s, slot & kDirSlotMask) + cell_index(x, y));
        const double dist = (w & kDmValid) ? mul_rn(sqrt((double)dm_sqdist(w)), resolution) : dmax;
        acc += mul_rn(dist, dist);
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double v = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += part[w];
        out[blockIdx.x] = sqrt(v / (double)scan.n_beams);
    }
}

__global__ void k_distance(StoreView s, int set, int particle, const double* __restrict__ pts, int n, double resolution, uint32_t max_sqdist,
                           double* __restrict__ dist, double* __restrict__ grad)
{
    const int32_t* d = dir_of(s, set, particle, kMapDm);
    const double scale = 1.0 / resolution;
    const double dmax  = mul_rn(sqrt((double)max_sqdist), resolution);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double mx = w2m_nocast(pts[3 * i], scale), my = w2m_nocast(pts[3 * i + 1], scale);
        const uint32_t dx = (uint32_t)mx, dy = (uint32_t)my;
        double v[4];
        for (int k = 0; k < 4; ++k) {
            uint32_t x = dx + (k & 1), y = dy + (k >> 1);
            int di = dir_index(s.window, x, y);
            int slot = di < 0 ? -1 : d[di];
            uint32_t w = slot < 0 ? 0u : __ldcg(patch_ptr(s, slot & kDirSlotMask) + cell_index(x, y));
            v[k] = (w & kDmValid) ? mul_rn(sqrt((double)dm_sqdist(w)), resolution) : dmax;
        }
        BeamEval e = bilinear(v, add_rn(mx, -(double)dx), add_rn(my, -(double)dy), scale, 0, 0);
        dist[i] = e.dist;
        if (grad) {
            grad[3 * i]     = e.gx;
            grad[3 * i + 1] = e.gy;
            grad[3 * i + 2] = 0.0;
        }
    }
}

// ==================================================================================================
// k_render_scans: posed scans cast into ONE frequency map (GraphSlam2D::generateOccupancyMap, graph_slam2d.cpp:131-164)
// ==================================================================================================
// One CTA per scan, lane = beam: the lanes of a warp walk angularly adjacent beams in lock step, so the reductions of one
// step fall into neighbouring cells.  Every update of a render is a counter increment, so there is no ordered path: no log,
// no replay, no candidate bitmaps.  kMark: the first pass only marks the directory entries of the touched cells (one byte
// each, written when the walk enters another patch), so that exactly the reference's patch set gets allocated before the
// counting pass; the counting pass walks the same cells and adds fire-and-forget reductions (hits: a returning add, see touch).
constexpr int kRenderThreads = 256;

template <bool kMark>
__global__ void __launch_bounds__(kRenderThreads) k_render_scans(StoreView s, int set, RenderParams p)
{
    __shared__ Affine tf;
    if (threadIdx.x == 0) tf = compose_tf(p.states[blockIdx.x], p.moving[blockIdx.x]);   // the transform of Slam2D's map update
    __syncthreads();
    const int32_t* dir = dir_of(s, set, 0, kMapOcc);
    const DirWindow win = s.window;
    const uint32_t bx0 = (uint32_t)win.base_px << kPatchLog2, by0 = (uint32_t)win.base_py << kPatchLog2;
    const uint32_t side = (uint32_t)win.dim << kPatchLog2;
    int log2dim = 0;
    while ((1 << (log2dim + 1)) <= win.dim) ++log2dim;
    ScanParams sp{};   // no truncation, no lidar-odometry rays: hit = tf * p, ray start = tf.translation()
    sp.scale = p.scale;
    uint32_t err = 0;
    unsigned long long cells = 0;
    int last_di = -1;
    uint32_t* base = nullptr;   // patch of last_di (counting pass); null: not allocated (the pool ran dry, reported)
    auto touch = [&](uint32_t P, uint32_t inc) {
        const int di = (int)packed_dir_index(P, log2dim);
        if (di != last_di) {
            last_di = di;
            if (kMark) {
                if (!p.marks[di]) p.marks[di] = 1;
            } else {
                const int e = __ldg(dir + di);
                base = e < 0 ? nullptr : patch_ptr(s, e & kDirSlotMask);
            }
        }
        if (kMark || !base) return;
        uint32_t* cell = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(base) + packed_cell_offset(P));
        if (inc == kOccHitInc) {
            // a hit (one touch in a few hundred) returns the old word: the hit that finds `occupied` at 0xFFFF wraps it, and its
            // carry into `visited` is taken back (adding 0xFFFF0000 leaves the low half alone; the adds of a cell commute)
            if (occ_occupied(atomicAdd(cell, kOccHitInc)) == 0xFFFFu)
                asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(cell), "r"(0u - kOccMissInc) : "memory");
        } else {
            asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(cell), "r"(inc) : "memory");
        }
        ++cells;
    };
    const int64_t b0 = p.offsets[blockIdx.x], b1 = p.offsets[blockIdx.x + 1];
    for (int64_t b = b0 + threadIdx.x; b < b1; b += blockDim.x) {
        const double pt[3] = {__ldg(p.points + 3 * b), __ldg(p.points + 3 * b + 1), __ldg(p.points + 3 * b + 2)};
        const BeamCells bc = beam_cells(tf, sp, pt);
        const uint32_t fx = bc.from[0] - bx0, fy = bc.from[1] - by0, tx = bc.to[0] - bx0, ty = bc.to[1] - by0;
        if ((fx | fy | tx | ty) >= side) {   // the beam leaves the directory window: reported, nothing is written
            err |= kErrWindow;
            continue;
        }
        touch(tx | (ty << 16), kOccHitInc);   // setOccupied(tf * p)
        if (!p.full) continue;
        if (bc.from[2] == bc.to[2]) {          // planar beam: the 2-axis form of computeRay (every 2-D scan)
            SegWalk w;
            w.init(fx, fy, tx, ty, 0, 1 << 30);
            while (w.next()) touch(w.P, kOccMissInc);
        } else {                               // tilted sensor: the 3-axis walk
            RayWalk3 w(bc);
            while (w.next()) touch((w.x - bx0) | ((w.y - by0) << 16), kOccMissInc);
        }
    }
    err = __reduce_or_sync(0xffffffffu, err);
    if ((threadIdx.x & 31) == 0 && err) atomicOr(s.status, err);
    if (!kMark) {
        for (int o = 16; o > 0; o >>= 1) cells += __shfl_xor_sync(0xffffffffu, cells, o);
        if ((threadIdx.x & 31) == 0 && cells) atomicAdd(p.cells, cells);
    }
}

// one warp per directory entry: a zeroed patch for every marked entry that has none (Map::get mutable, map.cpp:400-408)
__global__ void k_render_alloc(StoreView s, int set, const uint8_t* __restrict__ marks)
{
    const int lane = threadIdx.x & 31;
    const int di   = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (di >= s.window.dim * s.window.dim || !marks[di]) return;
    int32_t* dir = dir_of(s, set, 0, kMapOcc);
    if (dir[di] >= 0) return;
    int ns = 0;
    if (lane == 0) {
        ns = alloc_slot(s);
        if (ns >= 0) atomicAdd((unsigned long long*)&s.counters[0], 1ull);
    }
    ns = __shfl_sync(0xffffffffu, ns, 0);
    if (ns < 0) return;
    warp_zero_patch(patch_ptr(s, ns), lane);
    fbits_ptr(s, ns)[lane] = 0u;
    kbits_ptr(s, ns)[lane] = 0u;
    if (lane == 0) dir[di] = ns | kDirOwn;
}

// one warp per directory entry touched by the render: known |= (word != 0) (every touch went through Map::get, which sets the
// Container bit; a touched cell's word is 0 only when both counters wrapped back to 0, DESIGN.md §10), then the mark is cleared for
// the next render
__global__ void k_render_known(StoreView s, int set, uint8_t* __restrict__ marks)
{
    const int lane = threadIdx.x & 31;
    const int di   = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (di >= s.window.dim * s.window.dim || !marks[di]) return;
    const int e = dir_of(s, set, 0, kMapOcc)[di];
    if (e >= 0) {
        const uint32_t* cells = patch_ptr(s, e & kDirSlotMask);
        uint32_t* kb = kbits_ptr(s, e & kDirSlotMask);
        for (int row = 0; row < kPatchLen; ++row) {
            const uint32_t known = __ballot_sync(0xffffffffu, __ldcg(cells + row * kPatchLen + lane) != 0u);
            if (lane == 0 && known) kb[row] |= known;
        }
    }
    if (lane == 0) marks[di] = 0;
}

// FrequencyOccupancyMap::prune (frequency_occupancy_map.cpp:149-158) over every patch: cells visited once and occupied at most
// once go back to {0, 0}; their known bit stays
__global__ void k_prune_freq(StoreView s, int set)
{
    const int lane = threadIdx.x & 31;
    const int di   = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (di >= s.window.dim * s.window.dim) return;
    const int e = dir_of(s, set, 0, kMapOcc)[di];
    if (e < 0) return;
    uint32_t* cells = patch_ptr(s, e & kDirSlotMask);
    for (int row = 0; row < kPatchLen; ++row) {
        const uint32_t w = cells[row * kPatchLen + lane];
        if (occ_visited(w) == 1u && occ_occupied(w) <= 1u) cells[row * kPatchLen + lane] = 0u;
    }
}

}  // namespace

// ==================================================================================================
// host-side launch wrappers
// ==================================================================================================
size_t match_smem_bytes(int dir_dim, uint32_t max_sqdist)
{
    return (size_t)dir_dim * dir_dim * 4 + (size_t)(max_sqdist + 1) * 8 + ((sizeof(MatchShared) + 15) & ~(size_t)15) + (size_t)kNumSums * kMatchThreads * 8 + 16;
}
size_t raycast_smem_bytes(int dir_dim, const RayParams& rp)
{
    const int dim2 = dir_dim * dir_dim;
    const int n_groups = (rp.scan.n_beams + 31) / 32;
    const size_t beam_bytes = (size_t)n_groups * 32 * 16, ev_bytes = (size_t)rp.event_cap * 8;
    const size_t prob_extra = rp.prob_mode ? (size_t)dim2 * 4 + (size_t)((dim2 + 31) / 32) * 4 + 32 : 0;
    return (size_t)dim2 * 4 + (size_t)rp.log_cap * 8 + (beam_bytes > ev_bytes ? beam_bytes : ev_bytes) + (size_t)rp.cand_cap * 128 +
           (size_t)((dim2 + 31) / 32) * 8 + (size_t)(n_groups + 4) * 4 + (size_t)(rp.cand_cap + 4) * 2 + (size_t)dim2 * 4 + sizeof(RayShared) + 32 + prob_extra;
}
size_t brushfire_smem_bytes(int dir_dim, const BrushParams& bp)
{
    const int dim2 = dir_dim * dir_dim;
    return (size_t)dim2 * 4 + (size_t)(bp.lower_cap + bp.raise_cap + 4 + bp.event_cap) * 8 + 32 * 4 + 16 + 16;
}

// The dynamic shared-memory limit of a kernel is process-wide state, while engines of different configurations live side by side (a
// GraphSlam2D's inner Slam2D next to its global maps, a Loc2D next to a PFSlam2D): an engine only ever raises it.
template <typename Kernel>
static cudaError_t raise_smem_limit(Kernel* k, size_t bytes)
{
    cudaFuncAttributes a;
    cudaError_t e = cudaFuncGetAttributes(&a, k);
    if (e != cudaSuccess) return e;
    if ((size_t)a.maxDynamicSharedSizeBytes >= bytes) return cudaSuccess;
    return cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

cudaError_t configure_kernels(int dir_dim, uint32_t max_sqdist_limit, const RayParams& rp, const BrushParams& bp)
{
    cudaError_t e;
    e = raise_smem_limit(k_match, match_smem_bytes(dir_dim, max_sqdist_limit));
    if (e != cudaSuccess) return e;
    if (rp.prob_mode) e = raise_smem_limit(k_raycast<true>, raycast_smem_bytes(dir_dim, rp));
    else e = raise_smem_limit(k_raycast<false>, raycast_smem_bytes(dir_dim, rp));
    if (e != cudaSuccess) return e;
    e = raise_smem_limit(k_brushfire, brushfire_smem_bytes(dir_dim, bp));
    if (e != cudaSuccess) return e;
    e = raise_smem_limit(k_ray_setup, ray_setup_smem_bytes(dir_dim, rp.scan.n_beams > 4096 ? 4096 : rp.scan.n_beams));
    if (e != cudaSuccess) return e;
    e = raise_smem_limit(k_ray_pull<false>, ray_pull_smem_bytes(rp.scan.n_beams > 4096 ? 4096 : rp.scan.n_beams));
    if (e != cudaSuccess) return e;
    e = raise_smem_limit(k_ray_pull<true>, ray_pull_smem_bytes(rp.scan.n_beams > 4096 ? 4096 : rp.scan.n_beams));
    return e;
}

void launch_match(const StoreView& s, const MatchParams& mp, const SE2* d_states, MatchResult* d_results, int count, cudaStream_t st)
{
    if (count <= 0) return;
    // every thread evaluates ceil(n / threads) beams: choose the block so that the last round is (almost) full
    const int n = mp.scan.n_beams, rounds = (n + kMatchThreads - 1) / kMatchThreads;
    int threads = (((n + rounds - 1) / rounds) + 31) & ~31;
    threads = threads < 128 ? 128 : threads;
    k_match<<<count, threads, match_smem_bytes(s.window.dim, mp.max_sqdist), st>>>(s, mp, d_states, d_results);
}
void launch_raycast(const StoreView& s, const RayParams& rp, const SE2* d_states, uint64_t* d_events, MapUpdateStats* d_stats, int count,
                    cudaStream_t st)
{
    if (count <= 0) return;
    if (rp.prob_mode) k_raycast<true><<<count, kRayThreads, raycast_smem_bytes(s.window.dim, rp), st>>>(s, rp, d_states, d_events, d_stats);
    else k_raycast<false><<<count, kRayThreads, raycast_smem_bytes(s.window.dim, rp), st>>>(s, rp, d_states, d_events, d_stats);
}
size_t ray_setup_smem_bytes(int dir_dim, int n_beams) { return RaySetupLayout(n_beams, dir_dim * dir_dim).total; }
size_t ray_pull_smem_bytes(int n_beams) { return RayPullLayout(n_beams).total; }
void launch_raycast_pull(const StoreView& s, const RayParams& rp_in, const SE2* d_states, uint64_t* d_events, MapUpdateStats* d_stats, int count, int n_sms,
                         cudaStream_t st)
{
    if (count <= 0) return;
    RayParams rp = rp_in;
    // work units: enough of them to fill the machine several times over whatever the number of particles on this device
    int splits = (6 * n_sms + count - 1) / count;
    rp.pull.splits = splits < 1 ? 1 : (splits > 64 ? 64 : splits);
    k_ray_setup<<<count, kSetupThreads, ray_setup_smem_bytes(s.window.dim, rp.scan.n_beams), st>>>(s, rp, d_states, d_stats);
    const int units = count * rp.pull.splits;
    const int grid = units < n_sms * kPullCtasPerSm ? units : n_sms * kPullCtasPerSm;   // persistent: every CTA of eight warps resident
    const size_t smem = ray_pull_smem_bytes(rp.scan.n_beams);
    if (rp.prob_mode) k_ray_pull<true><<<grid, kPullWarps * 32, smem, st>>>(s, rp, count, d_events, d_stats);
    else k_ray_pull<false><<<grid, kPullWarps * 32, smem, st>>>(s, rp, count, d_events, d_stats);
}
void launch_brushfire(const StoreView& s, const BrushParams& bp, uint64_t* d_events, MapUpdateStats* d_stats, int count, cudaStream_t st)
{
    if (count <= 0) return;
    k_brushfire<<<count, kBrushThreads, brushfire_smem_bytes(s.window.dim, bp), st>>>(s, bp, d_events, d_stats);
}
void launch_copy_dirs(const StoreView& s, int src_set, int dst_set, const int32_t* d_idx, int dst_first, int count, cudaStream_t st)
{
    if (count <= 0) return;
    k_copy_dirs<<<dim3(count, 2), 256, 0, st>>>(s, src_set, dst_set, d_idx, dst_first);
}
void launch_release(const StoreView& s, int set, int first, int count, cudaStream_t st)
{
    if (count <= 0) return;
    k_release<<<dim3(count, s.n_kinds), 256, 0, st>>>(s, set, first);
}
void launch_merge_free(const StoreView& s, cudaStream_t st) { k_merge_free<<<1, 256, 0, st>>>(s); }
void launch_pack_results(const MatchResult* d_results, int n, double digest, double* d_out, cudaStream_t st)
{
    k_pack_results<<<(n + 127) / 128, 128, 0, st>>>(d_results, n, digest, d_out);
}
void launch_delete_patches(const StoreView& s, int set, int particle, const int32_t* d_list, int count, cudaStream_t st)
{
    if (count <= 0) return;
    k_delete_patches<<<count, 32, 0, st>>>(s, set, particle, d_list);
}
void launch_init_store(const StoreView& s, int n_sets, cudaStream_t st) { k_init_store<<<296, 256, 0, st>>>(s, n_sets); }
void launch_export(const StoreView& s, int set, int particle, int kind, uint32_t x0, uint32_t y0, int w, int h, uint32_t* d_out, uint8_t* d_present,
                   cudaStream_t st)
{
    int blocks = (w * h + 255) / 256;
    if (blocks > 1184) blocks = 1184;
    if (blocks < 1) blocks = 1;
    k_export<<<blocks, 256, 0, st>>>(s, set, particle, kind, x0, y0, w, h, d_out, d_present);
}
void launch_gather_cells(const StoreView& s, int set, int particle, int kind, const uint32_t* d_cells, int n, uint32_t* d_words, uint8_t* d_flags,
                         cudaStream_t st)
{
    if (n <= 0) return;
    k_gather_cells<<<(n + 255) / 256 < 592 ? (n + 255) / 256 : 592, 256, 0, st>>>(s, set, particle, kind, d_cells, n, d_words, d_flags);
}
void launch_export_bits(const StoreView& s, int plane, int set, int particle, uint32_t x0, uint32_t y0, int w, int h, uint8_t* d_out, cudaStream_t st)
{
    int blocks = (w * h + 255) / 256;
    if (blocks > 1184) blocks = 1184;
    if (blocks < 1) blocks = 1;
    k_export_bits<<<blocks, 256, 0, st>>>(s, plane, set, particle, x0, y0, w, h, d_out);
}
void launch_import(const StoreView& s, int set, int particle, int kind, uint32_t x0, uint32_t y0, int w, int h, const uint32_t* d_in, cudaStream_t st)
{
    int patches = (w / kPatchLen) * (h / kPatchLen);
    if (patches <= 0) return;
    k_import<<<(patches + 3) / 4, 128, 0, st>>>(s, set, particle, kind, x0, y0, w, h, d_in);
}
void launch_gather_patches(const StoreView& s, const int32_t* d_slots, int n, uint32_t* d_out, uint32_t* d_out_fbits, uint32_t* d_out_kbits,
                           cudaStream_t st)
{
    if (n <= 0) return;
    k_gather_patches<<<(n + 3) / 4, 128, 0, st>>>(s, d_slots, n, d_out, d_out_fbits, d_out_kbits);
}
size_t ckpt_scan_temp_bytes(int n_slots)
{
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const int32_t*)nullptr, (int32_t*)nullptr, n_slots);
    return bytes;
}
void launch_ckpt_compact(const StoreView& s, int set, const CkptScratch& c, cudaStream_t st, cudaEvent_t after_count)
{
    const size_t n_dir = (size_t)s.n_particles * s.n_kinds * s.window.dim * s.window.dim;
    const int dir_blocks = (int)std::min<size_t>((n_dir + 255) / 256, 4736), slot_blocks = std::min((s.n_slots + 255) / 256, 4736);
    k_ckpt_count<<<dir_blocks, 256, 0, st>>>(s, set, c.cnt, c.bad);
    if (after_count) cudaEventRecord(after_count, st);
    k_ckpt_mark<<<slot_blocks, 256, 0, st>>>(s, c.cnt, c.used, c.bad);
    size_t temp = c.temp_bytes;
    cub::DeviceScan::ExclusiveSum(c.temp, temp, c.used, c.new_id, s.n_slots, st);
    k_ckpt_list<<<slot_blocks, 256, 0, st>>>(s, c.used, c.new_id, c.list, c.ref);
    k_ckpt_remap<<<dir_blocks, 256, 0, st>>>(s, set, c.new_id, c.dirs);
}
void launch_scatter_patches(const StoreView& s, int set, int particle, int kind, const int32_t* d_entries, int n, const uint32_t* d_in,
                            const uint32_t* d_in_fbits, cudaStream_t st)
{
    if (n <= 0) return;
    k_scatter_patches<<<(n + 3) / 4, 128, 0, st>>>(s, set, particle, kind, d_entries, n, d_in, d_in_fbits);
}
void launch_sampling(const StoreView& s, int set, int particle, const double* d_points, const ScanParams& scan, const SE2& pose, const double* d_offsets,
                     int n_offsets, int stride, double resolution, uint32_t max_sqdist, double* d_out, cudaStream_t st)
{
    if (n_offsets <= 0) return;
    k_sampling<<<n_offsets, 128, 0, st>>>(s, set, particle, d_points, scan, pose, d_offsets, stride, resolution, max_sqdist, d_out);
}
void launch_match_error(const StoreView& s, int set, int particle0, bool shared_map, const double* d_points, const ScanParams& scan, const SE2* d_states, int count,
                        double resolution, uint32_t max_sqdist, double* d_out, cudaStream_t st)
{
    if (count <= 0) return;
    k_match_error<<<count, 256, 0, st>>>(s, set, particle0, shared_map ? 1 : 0, d_points, scan, d_states, resolution, max_sqdist, d_out);
}
void launch_distance(const StoreView& s, int set, int particle, const double* d_pts, int n, double resolution, uint32_t max_sqdist, double* d_dist,
                     double* d_grad, cudaStream_t st)
{
    if (n <= 0) return;
    int blocks = (n + 255) / 256;
    if (blocks > 1184) blocks = 1184;
    k_distance<<<blocks, 256, 0, st>>>(s, set, particle, d_pts, n, resolution, max_sqdist, d_dist, d_grad);
}
void launch_render_scans(const StoreView& s, int set, const RenderParams& p, int n_scans, cudaStream_t st)
{
    if (n_scans <= 0) return;
    const int dim2 = s.window.dim * s.window.dim, blocks = (dim2 + 7) / 8;   // one warp per directory entry
    k_render_scans<true><<<n_scans, kRenderThreads, 0, st>>>(s, set, p);
    k_render_alloc<<<blocks, 256, 0, st>>>(s, set, p.marks);
    k_render_scans<false><<<n_scans, kRenderThreads, 0, st>>>(s, set, p);
    k_render_known<<<blocks, 256, 0, st>>>(s, set, p.marks);
}
void launch_prune_freq(const StoreView& s, int set, cudaStream_t st)
{
    const int dim2 = s.window.dim * s.window.dim;
    k_prune_freq<<<(dim2 + 7) / 8, 256, 0, st>>>(s, set);
}

}  // namespace lama_b200
