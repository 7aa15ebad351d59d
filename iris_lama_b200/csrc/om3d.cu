// om3d.cu -- lama::FrequencyOccupancyMap and lama::ProbabilisticOccupancyMap with is3d = true on the device: point-cloud insertion
// (the loop body of GraphSlam2D::generateOccupancyMap, graph_slam2d.cpp:146-158), ordered per-cell setters, queries, prune, exports
// and 3-D .sdm files.
//
// Insertion, frequency maps.  Every update is a counter increment and increments commute, so the map is built as the 2-D render
// (k_render_scans) builds it:
//   1. k_om3_points<0> (mark): one thread per point, the lanes of a warp on consecutive points.  The thread walks its hit and its ray, checks
//      the window, marks the touched directory entries and counts its updates.  Nothing in the map is written yet: a window error
//      leaves it unchanged.
//   2. The host allocates the marked patches from the pool in ascending directory index (the reference's patch set); k_om3_zero
//      clears them.
//   3. k_om3_points<1> (count) walks again and adds fire-and-forget `red.global.add.u32` reductions.  A hit is a returning add: the hit that
//      finds `occupied` at 0xFFFF takes its carry out of `visited` back.
//   4. k_om3_known sets known |= (word != 0) over the marked entries.
// Insertion, log-odds maps.  Updates are clamped, so their order matters; they are replayed in the reference's order as the TSDM
// fusion does (tsdm.cu): per-point record counts (1 + ray cells) and an exclusive scan place the records in (cloud, point, step)
// order, step 0 being the hit.  The batch is cut at cloud boundaries into chunks of at most kRecordCap records; per chunk
// k_om3_points<2> (emit) writes the records and sets the known bits, a stable radix sort on the cell key groups them by cell (the op travels in
// the value), and k_om3_fold folds each run of equal keys in record order with prob_hit / prob_miss.
// apply() uses the same record -> sort -> fold path for both kinds, with the op's list index in the value.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "engine.h"
#include "om3d.h"
#include "om3d_core.h"
#include "sdm_io.h"

namespace lama_b200 {

namespace {

constexpr uint64_t kRecordCap = uint64_t(1) << 24;   // records of one sort chunk (a longer single cloud gets a chunk of its own)
constexpr int kMaxDim = 2048;                         // patches per window axis
constexpr int kThreads = 256;
constexpr uint64_t kUniversalConstant = 2642244ull;   // map.h:68

struct View {
    const int32_t* dir;   // slot of each directory entry, -1 = absent
    uint32_t* cells;      // pool: kOm3Cells words per slot
    uint32_t* known;      // pool: kOm3KnownWords words per slot
    TsdmWindow w;
};

__device__ __forceinline__ size_t pool_index(int slot, uint32_t ci) { return ((size_t)slot << kOm3Log2Cells) | ci; }
__device__ __forceinline__ uint32_t cell_index(uint32_t x, uint32_t y, uint32_t z) { return tsdm_cell_index(x, y, z, 1); }

struct InsertParams {
    const double* pts;
    const int64_t* offsets;   // n_clouds + 1
    const Affine* tf;         // per cloud: Translation(sensor_origin_) * sensor_orientation_
    int n_clouds;
    int64_t p0, p1;           // the points of this pass
    double scale;
    int full;
    uint64_t* counts;         // per point: records (1 + ray cells)
    const uint64_t* offs;     // exclusive scan of counts
    uint64_t rec_base;
    uint32_t* rkeys;          // record: directory index << 15 | cell index
    uint32_t* rvals;          // record: op
    uint32_t* marks;          // per directory entry: touched by this batch
    uint32_t* status;
};

__device__ __forceinline__ int cloud_of(const int64_t* off, int n, int64_t p)
{
    int lo = 0, hi = n;   // the last cloud c with off[c] <= p
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (off[mid] <= p) lo = mid; else hi = mid;
    }
    return lo;
}

// kPass 0 (mark): window check, directory marks, record counts.  1 (count, frequency maps): counter reductions.  2 (emit, log-odds
// maps): known bits and records.  Every pass visits the cells of a point in the reference's order: the hit, then the ray from so.
template <int kPass>
__global__ void __launch_bounds__(kThreads) k_om3_points(InsertParams f, View v)
{
    const int64_t p = f.p0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= f.p1) return;
    const int c = cloud_of(f.offsets, f.n_clouds, p);
    const BeamCells b = om3_point_cells(f.tf[c], f.pts + 3 * p, f.scale);
    int last_di = -2;
    uint32_t* base = nullptr;
    uint64_t out = kPass == 2 ? f.offs[p] - f.rec_base : 0;
    bool bad = false;
    auto touch = [&](uint32_t x, uint32_t y, uint32_t z, uint32_t op) {
        const int di = tsdm_dir_index(v.w, x, y, z);
        if (kPass == 0) {
            if (di < 0) { bad = true; return; }
            if (di != last_di) {
                last_di = di;
                if (!f.marks[di]) f.marks[di] = 1;
            }
            return;
        }
        const uint32_t ci = cell_index(x, y, z);
        const int slot = v.dir[di];
        if (kPass == 2) {
            const size_t g = pool_index(slot, ci);
            atomicOr(&v.known[g >> 5], 1u << (g & 31));
            f.rkeys[out] = ((uint32_t)di << kOm3Log2Cells) | ci;
            f.rvals[out] = op;
            ++out;
            return;
        }
        if (di != last_di) {
            last_di = di;
            base = v.cells + ((size_t)slot << kOm3Log2Cells);
        }
        uint32_t* cell = base + ci;
        if (op == kOm3SetOccupied) {
            // the 65 536th hit of a cell carries out of `occupied` into `visited`: the hit that finds 0xFFFF takes it back
            if (occ_occupied(atomicAdd(cell, kOccHitInc)) == 0xFFFFu)
                asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(cell), "r"(0u - kOccMissInc) : "memory");
        } else {
            asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(cell), "r"(kOccMissInc) : "memory");
        }
    };
    touch(b.to[0], b.to[1], b.to[2], kOm3SetOccupied);   // setOccupied(tf * p)
    if (f.full) {                                        // setFree on computeRay(so, w2m(hit))
        RayWalk3 w(b);
        while (w.next() && !bad) touch(w.x, w.y, w.z, kOm3SetFree);
    }
    if (kPass == 0) {
        if (bad) atomicOr(f.status, kErrWindow);
        f.counts[p] = om3_point_records(b, f.full != 0);
    }
}

// one block per directory entry marked by the batch: known |= (word != 0) (every touch went through Map::get, which sets the
// Container bit; a touched cell whose two counters both wrapped to 0 in one batch is missed, DESIGN.md §10)
__global__ void __launch_bounds__(kThreads) k_om3_known(View v, const uint32_t* __restrict__ marks)
{
    const int di = blockIdx.x;
    if (!marks[di]) return;
    const int slot = v.dir[di];
    const uint32_t* cells = v.cells + ((size_t)slot << kOm3Log2Cells);
    uint32_t* kb = v.known + (size_t)slot * kOm3KnownWords;
    const int lane = threadIdx.x & 31;
    for (int row = threadIdx.x >> 5; row < kOm3KnownWords; row += kThreads / 32) {
        const uint32_t k = __ballot_sync(0xffffffffu, __ldcg(cells + row * 32 + lane) != 0u);
        if (lane == 0 && k) kb[row] |= k;
    }
}

__global__ void k_om3_zero(const int32_t* slots, int n, View v)
{
    const size_t total = (size_t)n << kOm3Log2Cells;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t g = pool_index(slots[i >> kOm3Log2Cells], (uint32_t)(i & (kOm3Cells - 1)));
        v.cells[g] = 0u;
        if ((g & 31) == 0) v.known[g >> 5] = 0u;
    }
}

__global__ void k_om3_gather_bounds(const uint64_t* offs, const int64_t* idx, int n, uint64_t* out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = offs[idx[i]];
}

// apply(): kEmit = false: window check and marks; true: known bits and records (value = list index << 2 | op)
template <bool kEmit>
__global__ void __launch_bounds__(kThreads) k_om3_apply(const uint32_t* __restrict__ xyz, const uint8_t* __restrict__ ops, int n, View v,
                                                        uint32_t* marks, uint32_t* status, uint32_t* rkeys, uint32_t* rvals)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    const int di = tsdm_dir_index(v.w, x, y, z);
    if (!kEmit) {
        if (di < 0) atomicOr(status, kErrWindow);
        else if (!marks[di]) marks[di] = 1;
        return;
    }
    const uint32_t ci = cell_index(x, y, z);
    const size_t g = pool_index(v.dir[di], ci);
    atomicOr(&v.known[g >> 5], 1u << (g & 31));
    rkeys[i] = ((uint32_t)di << kOm3Log2Cells) | ci;
    rvals[i] = ((uint32_t)i << 2) | ops[i];
}

// one thread per run of equal cell keys: the run's ops in record order, from the stored cell.  kApply: changed[value >> 2].
template <bool kApply>
__global__ void __launch_bounds__(kThreads) k_om3_fold(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint64_t n, View v,
                                                       int kind, ProbParams pp, uint8_t* changed)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t k = keys[i];
    if (i > 0 && keys[i - 1] == k) return;
    const size_t g = pool_index(v.dir[k >> kOm3Log2Cells], k & (kOm3Cells - 1));
    uint32_t word = v.cells[g];
    for (uint64_t j = i; j < n && keys[j] == k; ++j) {
        const uint32_t r = vals[j];
        const bool ch = om3_op(kind, word, r & 3u, pp);
        if (kApply) changed[r >> 2] = ch;
    }
    v.cells[g] = word;
}

// the cells the const get() returns (map.cpp:414-455, container.h:119-123): word and present (patch allocated, known bit set)
__global__ void __launch_bounds__(kThreads) k_om3_gather(const uint32_t* __restrict__ xyz, int n, View v, uint32_t* words, uint8_t* present)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    const int di = tsdm_dir_index(v.w, x, y, z);
    const int slot = di < 0 ? -1 : v.dir[di];
    uint32_t w = 0;
    bool k = false;
    if (slot >= 0) {
        const size_t g = pool_index(slot, cell_index(x, y, z));
        k = (v.known[g >> 5] >> (g & 31)) & 1u;
        w = k ? v.cells[g] : 0u;
    }
    words[i] = w;
    present[i] = k;
}

__global__ void k_om3_export(View v, uint32_t x0, uint32_t y0, uint32_t z0, int w, int h, int dd, uint32_t* words, uint8_t* known)
{
    const size_t n = (size_t)w * h * dd;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t x = x0 + (uint32_t)(i % w), y = y0 + (uint32_t)((i / w) % h), z = z0 + (uint32_t)(i / ((size_t)w * h));
        const int di = tsdm_dir_index(v.w, x, y, z);
        const int slot = di < 0 ? -1 : v.dir[di];
        uint32_t c = 0;
        uint8_t k = 0;
        if (slot >= 0) {
            const size_t g = pool_index(slot, cell_index(x, y, z));
            c = v.cells[g];
            k = (v.known[g >> 5] >> (g & 31)) & 1u;
        }
        words[i] = c;
        known[i] = k;
    }
}

// FrequencyOccupancyMap::prune (frequency_occupancy_map.cpp:149-158) over the known cells of the first n_slots pool slots
__global__ void k_om3_prune(View v, int n_slots)
{
    const size_t total = (size_t)n_slots << kOm3Log2Cells;
    for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
        if (!((v.known[g >> 5] >> (g & 31)) & 1u)) continue;
        const uint32_t w = v.cells[g];
        const uint32_t p = om3_prune(w);
        if (p != w) v.cells[g] = p;
    }
}

inline unsigned blocks_for(uint64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

}  // namespace

// ---- host side ----------------------------------------------------------------------------------------------------------------
struct OccMap3Dev::Impl {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false, timing = false;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    int kind = kOm3Frequency;
    double resolution = 0, scale = 0;
    ProbParams pp{};
    TsdmWindow win{};
    int ndir = 0, pool = 0, used = 0, end_bit = 0;
    std::vector<int32_t> h_dir;
    int32_t* dir = nullptr;
    uint32_t* cells = nullptr;
    uint32_t* known = nullptr;
    uint32_t* status = nullptr;
    uint32_t* marks = nullptr;
    double ms[3] = {0, 0, 0};
    uint64_t launches[3] = {0, 0, 0};
    struct Buf { void* p = nullptr; size_t bytes = 0; };
    Buf pts, off, tf, counts, offs, bound, slots, rk[2], rv[2], temp, qin, qout, qflag, ops, changed;

    View view() const { return View{dir, cells, known, win}; }
    cudaError_t ensure(Buf& b, size_t bytes)
    {
        if (b.bytes >= bytes) return cudaSuccess;
        if (b.p) cudaFree(b.p);
        b.p = nullptr;
        b.bytes = 0;
        cudaError_t e = cudaMalloc(&b.p, bytes);
        if (e == cudaSuccess) b.bytes = bytes;
        return e;
    }
    ~Impl()
    {
        cudaSetDevice(device);
        if (stream) cudaStreamSynchronize(stream);
        Buf* all[] = {&pts, &off, &tf, &counts, &offs, &bound, &slots, &rk[0], &rk[1], &rv[0], &rv[1], &temp, &qin, &qout, &qflag, &ops, &changed};
        for (Buf* b : all)
            if (b->p) cudaFree(b->p);
        for (void* p : {(void*)dir, (void*)cells, (void*)known, (void*)status, (void*)marks})
            if (p) cudaFree(p);
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
        if (own_stream && stream) cudaStreamDestroy(stream);
    }
    // allocates the marked entries that have no patch (ascending directory index) and zeroes them; LAMA_ERR_POOL before any change
    int alloc_marked(const std::vector<uint32_t>& marks, std::string& err, uint64_t& launch_count)
    {
        std::vector<int32_t> fresh;
        for (int i = 0; i < ndir; ++i)
            if (marks[i] && h_dir[i] < 0) fresh.push_back(i);
        if ((int64_t)used + (int64_t)fresh.size() > pool) { err = "the patch pool is exhausted (raise pool_slots)"; return LAMA_ERR_POOL; }
        if (fresh.empty()) return LAMA_OK;
        std::vector<int32_t> sl(fresh.size());
        for (size_t i = 0; i < fresh.size(); ++i) h_dir[fresh[i]] = sl[i] = used++;
        cudaError_t e = ensure(slots, sl.size() * 4);
        if (e == cudaSuccess) e = cudaMemcpyAsync(slots.p, sl.data(), sl.size() * 4, cudaMemcpyHostToDevice, stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dir, h_dir.data(), (size_t)ndir * 4, cudaMemcpyHostToDevice, stream);
        if (e != cudaSuccess) { err = std::string("patch allocation: ") + cudaGetErrorString(e); return LAMA_ERR_CUDA; }
        k_om3_zero<<<std::min<uint64_t>(4096, blocks_for((uint64_t)sl.size() << kOm3Log2Cells)), kThreads, 0, stream>>>((const int32_t*)slots.p,
                                                                                                                      (int)sl.size(), view());
        launch_count += 1;
        return LAMA_OK;
    }
    // directory index -> the patch's anchor cell
    void anchor(int i, uint32_t a[3]) const
    {
        const int p[3] = {i % win.dim[0], (i / win.dim[0]) % win.dim[1], i / (win.dim[0] * win.dim[1])};
        for (int k = 0; k < 3; ++k) a[k] = (uint32_t)(win.base[k] + p[k]) << kPatchLog2;
    }
};

#define OM_TRY(expr)                                                                                        \
    do {                                                                                                    \
        cudaError_t _e = (expr);                                                                            \
        if (_e != cudaSuccess) { err_ = std::string(#expr) + ": " + cudaGetErrorString(_e); return LAMA_ERR_CUDA; } \
    } while (0)

OccMap3Dev* OccMap3Dev::create(double resolution, uint32_t patch_size, int kind, const double center[3], const int32_t window[3],
                               const DeviceOptions& dev, std::string& err)
{
    if (!(resolution > 0)) { err = "resolution must be positive"; return nullptr; }
    if (patch_size != (uint32_t)kPatchLen) { err = "patch_size must be 32 (the device patch layout)"; return nullptr; }
    if (kind != kOm3Frequency && kind != kOm3LogOdds) { err = "kind must be 0 (frequency) or 1 (log-odds)"; return nullptr; }
    int32_t dim[3] = {8, 8, 4};
    if (window) for (int k = 0; k < 3; ++k) dim[k] = window[k];
    for (int k = 0; k < 3; ++k)
        if (dim[k] < 1 || dim[k] > kMaxDim) { err = "window must be 1..2048 patches per axis"; return nullptr; }
    const int64_t ndir = (int64_t)dim[0] * dim[1] * dim[2];
    if (ndir > kOm3MaxEntries) { err = "window has more than 65536 patches"; return nullptr; }
    const int pool = dev.pool_slots > 0 ? dev.pool_slots : (int)ndir;

    OccMap3Dev* t = new OccMap3Dev();
    t->d_ = new Impl();
    Impl& d = *t->d_;
    d.device = dev.device;
    d.timing = dev.timing != 0;
    d.kind = kind;
    d.resolution = resolution;
    d.scale = 1.0 / resolution;
    {   // ProbabilisticOccupancyMap's constructor (probabilistic_occupancy_map.cpp:43-60): float logods(), stored as doubles
        auto logods = [](float prob) -> float { return (float)std::log(prob / (1.0 - prob)); };
        d.pp.miss      = logods(0.4f);
        d.pp.hit       = logods(0.7f);
        d.pp.clamp_min = logods(0.12f);
        d.pp.clamp_max = logods(0.97f);
        d.pp.thresh    = 0.0 * logods(0.5f);
    }
    d.win.is3d = 1;
    for (int k = 0; k < 3; ++k) {
        d.win.dim[k] = dim[k];
        const double c = center ? center[k] : 0.0;
        d.win.base[k] = (int32_t)(w2m(c, d.scale) >> kPatchLog2) - dim[k] / 2;
    }
    d.ndir = (int)ndir;
    d.pool = pool;
    d.end_bit = kOm3Log2Cells;
    while ((1ll << (d.end_bit - kOm3Log2Cells)) < ndir) ++d.end_bit;
    d.h_dir.assign((size_t)ndir, -1);
    auto bail = [&](const std::string& m) -> OccMap3Dev* { err = m; delete t; return nullptr; };
#define OM_NEW(expr)                                                                          \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) return bail(std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)
    OM_NEW(cudaSetDevice(dev.device));
    if (dev.stream) {
        d.stream = reinterpret_cast<cudaStream_t>(dev.stream);
    } else {
        OM_NEW(cudaStreamCreateWithFlags(&d.stream, cudaStreamNonBlocking));
        d.own_stream = true;
    }
    OM_NEW(cudaEventCreate(&d.ev[0]));
    OM_NEW(cudaEventCreate(&d.ev[1]));
    OM_NEW(cudaMalloc((void**)&d.dir, (size_t)ndir * 4));
    OM_NEW(cudaMalloc((void**)&d.marks, (size_t)ndir * 4));
    OM_NEW(cudaMalloc((void**)&d.cells, (size_t)pool * kOm3Cells * 4));
    OM_NEW(cudaMalloc((void**)&d.known, (size_t)pool * kOm3KnownWords * 4));
    OM_NEW(cudaMalloc((void**)&d.status, 4));
    OM_NEW(cudaMemcpyAsync(d.dir, d.h_dir.data(), (size_t)ndir * 4, cudaMemcpyHostToDevice, d.stream));
    OM_NEW(cudaStreamSynchronize(d.stream));
#undef OM_NEW
    return t;
}

OccMap3Dev::~OccMap3Dev() { delete d_; }

int OccMap3Dev::kind() const { return d_->kind; }
double OccMap3Dev::resolution() const { return d_->resolution; }

void OccMap3Dev::kernel_times(double ms[3], uint64_t launches[3]) const
{
    for (int k = 0; k < 3; ++k) {
        if (ms) ms[k] = d_->ms[k];
        if (launches) launches[k] = d_->launches[k];
    }
}

int OccMap3Dev::insert_point_clouds(const double* pts, const int64_t* offsets, int n_clouds, const double* origins, const double* quats, bool full,
                                    uint64_t* cells)
{
    Impl& d = *d_;
    if (cells) *cells = 0;
    if (n_clouds < 0) { err_ = "negative number of clouds"; return LAMA_ERR_ARG; }
    if (n_clouds == 0) return LAMA_OK;
    if (!offsets || offsets[0] != 0) { err_ = "offsets must start at 0"; return LAMA_ERR_ARG; }
    for (int k = 0; k < n_clouds; ++k)
        if (offsets[k + 1] < offsets[k]) { err_ = "offsets must not decrease"; return LAMA_ERR_ARG; }
    const int64_t n_pts = offsets[n_clouds];
    if (n_pts == 0) return LAMA_OK;
    if (!pts) { err_ = "null points"; return LAMA_ERR_ARG; }
    if (n_pts >= (int64_t)1 << 40) { err_ = "too many points"; return LAMA_ERR_ARG; }
    OM_TRY(cudaSetDevice(d.device));
    if (d.timing) OM_TRY(cudaEventRecord(d.ev[0], d.stream));
    std::vector<Affine> tf((size_t)n_clouds);
    for (int k = 0; k < n_clouds; ++k) {
        const MovingTf m = moving_tf(origins ? origins + 3 * k : nullptr, quats ? quats + 4 * k : nullptr);
        std::memcpy(tf[k].l, m.l, sizeof(m.l));
        std::memcpy(tf[k].t, m.t, sizeof(m.t));
    }
    OM_TRY(d.ensure(d.pts, (size_t)n_pts * 24));
    OM_TRY(d.ensure(d.off, (size_t)(n_clouds + 1) * 8));
    OM_TRY(d.ensure(d.tf, (size_t)n_clouds * sizeof(Affine)));
    OM_TRY(d.ensure(d.counts, (size_t)(n_pts + 1) * 8));
    OM_TRY(d.ensure(d.offs, (size_t)(n_pts + 1) * 8));
    OM_TRY(d.ensure(d.bound, (size_t)(n_clouds + 1) * 8));
    OM_TRY(cudaMemcpyAsync(d.pts.p, pts, (size_t)n_pts * 24, cudaMemcpyHostToDevice, d.stream));
    OM_TRY(cudaMemcpyAsync(d.off.p, offsets, (size_t)(n_clouds + 1) * 8, cudaMemcpyHostToDevice, d.stream));
    OM_TRY(cudaMemcpyAsync(d.tf.p, tf.data(), (size_t)n_clouds * sizeof(Affine), cudaMemcpyHostToDevice, d.stream));
    OM_TRY(cudaMemsetAsync(d.status, 0, 4, d.stream));
    OM_TRY(cudaMemsetAsync(d.marks, 0, (size_t)d.ndir * 4, d.stream));
    OM_TRY(cudaMemsetAsync((uint64_t*)d.counts.p + n_pts, 0, 8, d.stream));

    const View v0 = d.view();
    InsertParams f{};
    f.pts = (const double*)d.pts.p;
    f.offsets = (const int64_t*)d.off.p;
    f.tf = (const Affine*)d.tf.p;
    f.n_clouds = n_clouds;
    f.p0 = 0;
    f.p1 = n_pts;
    f.scale = d.scale;
    f.full = full ? 1 : 0;
    f.counts = (uint64_t*)d.counts.p;
    f.offs = (const uint64_t*)d.offs.p;
    f.marks = d.marks;
    f.status = d.status;

    // 1. window check, marks, record counts; the map is not touched
    k_om3_points<0><<<blocks_for(n_pts), kThreads, 0, d.stream>>>(f, v0);
    d.launches[0] += 1;
    OM_TRY(cudaGetLastError());
    uint32_t status = 0;
    OM_TRY(cudaMemcpyAsync(&status, d.status, 4, cudaMemcpyDeviceToHost, d.stream));
    std::vector<uint32_t> marks((size_t)d.ndir);
    OM_TRY(cudaMemcpyAsync(marks.data(), d.marks, (size_t)d.ndir * 4, cudaMemcpyDeviceToHost, d.stream));
    OM_TRY(cudaStreamSynchronize(d.stream));
    if (status & kErrWindow) { err_ = "a hit or ray cell lies outside the directory window"; return LAMA_ERR_WINDOW; }

    // 2. allocate the marked patches, ascending directory index
    int rc = d.alloc_marked(marks, err_, d.launches[0]);
    if (rc != LAMA_OK) return rc;
    const View v = d.view();

    // 3. record offsets (their total is the number of cell updates)
    size_t scan_bytes = 0;
    OM_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint64_t*)d.counts.p, (uint64_t*)d.offs.p, (int64_t)(n_pts + 1), d.stream));
    OM_TRY(d.ensure(d.temp, scan_bytes));
    OM_TRY(cub::DeviceScan::ExclusiveSum(d.temp.p, scan_bytes, (const uint64_t*)d.counts.p, (uint64_t*)d.offs.p, (int64_t)(n_pts + 1), d.stream));
    k_om3_gather_bounds<<<blocks_for(n_clouds + 1), kThreads, 0, d.stream>>>((const uint64_t*)d.offs.p, f.offsets, n_clouds + 1, (uint64_t*)d.bound.p);
    std::vector<uint64_t> bound((size_t)n_clouds + 1);
    OM_TRY(cudaMemcpyAsync(bound.data(), d.bound.p, bound.size() * 8, cudaMemcpyDeviceToHost, d.stream));
    OM_TRY(cudaStreamSynchronize(d.stream));
    d.launches[0] += 2;

    if (d.kind == kOm3Frequency) {
        // 4f. counter reductions, then the known plane of the touched patches
        k_om3_points<1><<<blocks_for(n_pts), kThreads, 0, d.stream>>>(f, v);
        k_om3_known<<<d.ndir, kThreads, 0, d.stream>>>(v, d.marks);
        d.launches[0] += 2;
    } else {
        // 4p. per chunk of whole clouds: records, stable sort on the cell key, one fold per cell
        for (int c0 = 0; c0 < n_clouds;) {
            int c1 = c0 + 1;
            while (c1 < n_clouds && bound[c1 + 1] - bound[c0] <= kRecordCap) ++c1;
            const uint64_t nrec = bound[c1] - bound[c0];
            if (nrec > 0) {
                for (int b = 0; b < 2; ++b) {
                    OM_TRY(d.ensure(d.rk[b], nrec * 4));
                    OM_TRY(d.ensure(d.rv[b], nrec * 4));
                }
                f.p0 = offsets[c0];
                f.p1 = offsets[c1];
                f.rec_base = bound[c0];
                f.rkeys = (uint32_t*)d.rk[0].p;
                f.rvals = (uint32_t*)d.rv[0].p;
                k_om3_points<2><<<blocks_for((uint64_t)(f.p1 - f.p0)), kThreads, 0, d.stream>>>(f, v);
                size_t sort_bytes = 0;
                OM_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t*)d.rk[0].p, (uint32_t*)d.rk[1].p, (const uint32_t*)d.rv[0].p,
                                                       (uint32_t*)d.rv[1].p, (int64_t)nrec, 0, d.end_bit, d.stream));
                OM_TRY(d.ensure(d.temp, sort_bytes));
                OM_TRY(cub::DeviceRadixSort::SortPairs(d.temp.p, sort_bytes, (const uint32_t*)d.rk[0].p, (uint32_t*)d.rk[1].p, (const uint32_t*)d.rv[0].p,
                                                       (uint32_t*)d.rv[1].p, (int64_t)nrec, 0, d.end_bit, d.stream));
                k_om3_fold<false><<<blocks_for(nrec), kThreads, 0, d.stream>>>((const uint32_t*)d.rk[1].p, (const uint32_t*)d.rv[1].p, nrec, v, d.kind,
                                                                              d.pp, nullptr);
                d.launches[0] += 3;
            }
            c0 = c1;
        }
    }
    OM_TRY(cudaGetLastError());
    if (d.timing) OM_TRY(cudaEventRecord(d.ev[1], d.stream));
    OM_TRY(cudaStreamSynchronize(d.stream));
    if (d.timing) {
        float t = 0;
        OM_TRY(cudaEventElapsedTime(&t, d.ev[0], d.ev[1]));
        d.ms[0] += t;
    }
    if (cells) *cells = bound[n_clouds];
    return LAMA_OK;
}

int OccMap3Dev::apply(const uint32_t* cells_xyz, const uint8_t* ops, int n, uint8_t* changed)
{
    Impl& d = *d_;
    if (n < 0 || (n > 0 && (!cells_xyz || !ops))) { err_ = "null argument"; return LAMA_ERR_ARG; }
    if (n == 0) return LAMA_OK;
    if (n >= (1 << 30)) { err_ = "too many ops"; return LAMA_ERR_ARG; }
    for (int i = 0; i < n; ++i)
        if (ops[i] > kOm3SetUnknown) { err_ = "op must be 0 (setFree), 1 (setOccupied) or 2 (setUnknown)"; return LAMA_ERR_ARG; }
    OM_TRY(cudaSetDevice(d.device));
    if (d.timing) OM_TRY(cudaEventRecord(d.ev[0], d.stream));
    OM_TRY(d.ensure(d.qin, (size_t)n * 12));
    OM_TRY(d.ensure(d.ops, (size_t)n));
    OM_TRY(d.ensure(d.changed, (size_t)n));
    for (int b = 0; b < 2; ++b) {
        OM_TRY(d.ensure(d.rk[b], (size_t)n * 4));
        OM_TRY(d.ensure(d.rv[b], (size_t)n * 4));
    }
    OM_TRY(cudaMemcpyAsync(d.qin.p, cells_xyz, (size_t)n * 12, cudaMemcpyHostToDevice, d.stream));
    OM_TRY(cudaMemcpyAsync(d.ops.p, ops, (size_t)n, cudaMemcpyHostToDevice, d.stream));
    OM_TRY(cudaMemsetAsync(d.status, 0, 4, d.stream));
    OM_TRY(cudaMemsetAsync(d.marks, 0, (size_t)d.ndir * 4, d.stream));
    const uint32_t* xyz = (const uint32_t*)d.qin.p;
    const uint8_t* dops = (const uint8_t*)d.ops.p;
    k_om3_apply<false><<<blocks_for(n), kThreads, 0, d.stream>>>(xyz, dops, n, d.view(), d.marks, d.status, nullptr, nullptr);
    d.launches[1] += 1;
    OM_TRY(cudaGetLastError());
    uint32_t status = 0;
    OM_TRY(cudaMemcpyAsync(&status, d.status, 4, cudaMemcpyDeviceToHost, d.stream));
    std::vector<uint32_t> marks((size_t)d.ndir);
    OM_TRY(cudaMemcpyAsync(marks.data(), d.marks, (size_t)d.ndir * 4, cudaMemcpyDeviceToHost, d.stream));
    OM_TRY(cudaStreamSynchronize(d.stream));
    if (status & kErrWindow) { err_ = "a cell lies outside the directory window"; return LAMA_ERR_WINDOW; }
    int rc = d.alloc_marked(marks, err_, d.launches[1]);
    if (rc != LAMA_OK) return rc;
    const View v = d.view();
    k_om3_apply<true><<<blocks_for(n), kThreads, 0, d.stream>>>(xyz, dops, n, v, nullptr, nullptr, (uint32_t*)d.rk[0].p, (uint32_t*)d.rv[0].p);
    size_t sort_bytes = 0;
    OM_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t*)d.rk[0].p, (uint32_t*)d.rk[1].p, (const uint32_t*)d.rv[0].p,
                                           (uint32_t*)d.rv[1].p, n, 0, d.end_bit, d.stream));
    OM_TRY(d.ensure(d.temp, sort_bytes));
    OM_TRY(cub::DeviceRadixSort::SortPairs(d.temp.p, sort_bytes, (const uint32_t*)d.rk[0].p, (uint32_t*)d.rk[1].p, (const uint32_t*)d.rv[0].p,
                                           (uint32_t*)d.rv[1].p, n, 0, d.end_bit, d.stream));
    k_om3_fold<true><<<blocks_for(n), kThreads, 0, d.stream>>>((const uint32_t*)d.rk[1].p, (const uint32_t*)d.rv[1].p, (uint64_t)n, v, d.kind, d.pp,
                                                              (uint8_t*)d.changed.p);
    d.launches[1] += 3;
    OM_TRY(cudaGetLastError());
    if (d.timing) OM_TRY(cudaEventRecord(d.ev[1], d.stream));
    if (changed) OM_TRY(cudaMemcpyAsync(changed, d.changed.p, (size_t)n, cudaMemcpyDeviceToHost, d.stream));
    OM_TRY(cudaStreamSynchronize(d.stream));
    if (d.timing) {
        float t = 0;
        OM_TRY(cudaEventElapsedTime(&t, d.ev[0], d.ev[1]));
        d.ms[1] += t;
    }
    return LAMA_OK;
}

int OccMap3Dev::query(const uint32_t* cells_xyz, int n, double* prob, uint8_t* flags)
{
    Impl& d = *d_;
    if (n < 0 || (n > 0 && !cells_xyz)) { err_ = "null argument"; return LAMA_ERR_ARG; }
    if (n == 0) return LAMA_OK;
    OM_TRY(cudaSetDevice(d.device));
    OM_TRY(d.ensure(d.qin, (size_t)n * 12));
    OM_TRY(d.ensure(d.qout, (size_t)n * 4));
    OM_TRY(d.ensure(d.qflag, (size_t)n));
    OM_TRY(cudaMemcpyAsync(d.qin.p, cells_xyz, (size_t)n * 12, cudaMemcpyHostToDevice, d.stream));
    if (d.timing) OM_TRY(cudaEventRecord(d.ev[0], d.stream));
    k_om3_gather<<<blocks_for(n), kThreads, 0, d.stream>>>((const uint32_t*)d.qin.p, n, d.view(), (uint32_t*)d.qout.p, (uint8_t*)d.qflag.p);
    d.launches[2] += 1;
    if (d.timing) OM_TRY(cudaEventRecord(d.ev[1], d.stream));
    OM_TRY(cudaGetLastError());
    std::vector<uint32_t> words((size_t)n);
    std::vector<uint8_t> present((size_t)n);
    OM_TRY(cudaMemcpyAsync(words.data(), d.qout.p, (size_t)n * 4, cudaMemcpyDeviceToHost, d.stream));
    OM_TRY(cudaMemcpyAsync(present.data(), d.qflag.p, (size_t)n, cudaMemcpyDeviceToHost, d.stream));
    OM_TRY(cudaStreamSynchronize(d.stream));
    if (d.timing) {
        float t = 0;
        OM_TRY(cudaEventElapsedTime(&t, d.ev[0], d.ev[1]));
        d.ms[2] += t;
    }
    // getProbability takes the host's expf, as the reference's float prob() does (probabilistic_occupancy_map.cpp:38-41)
    auto prob_of = [](float l) -> float { return 1.0 - 1.0 / (1.0 + std::exp(l)); };
    for (int i = 0; i < n; ++i) {
        if (flags) flags[i] = (uint8_t)om3_flags(d.kind, present[i] != 0, words[i], d.pp);
        if (!prob) continue;
        if (d.kind == kOm3Frequency) {   // frequency_occupancy_map.cpp:40-45,166-172
            const uint32_t occ = occ_occupied(words[i]), vis = occ_visited(words[i]);
            prob[i] = (!present[i] || vis == 0) ? 0.25 : ((double)occ) / ((double)vis);
        } else {                         // probabilistic_occupancy_map.cpp:169-175
            prob[i] = present[i] ? prob_of(om3_bits_float(words[i])) : prob_of((float)d.pp.thresh);
        }
    }
    return LAMA_OK;
}

int OccMap3Dev::prune()
{
    Impl& d = *d_;
    if (d.kind != kOm3Frequency) { err_ = "prune is a FrequencyOccupancyMap method"; return LAMA_ERR_ARG; }
    if (d.used == 0) return LAMA_OK;
    OM_TRY(cudaSetDevice(d.device));
    k_om3_prune<<<std::min<uint64_t>(8192, blocks_for((uint64_t)d.used << kOm3Log2Cells)), kThreads, 0, d.stream>>>(d.view(), d.used);
    OM_TRY(cudaGetLastError());
    OM_TRY(cudaStreamSynchronize(d.stream));
    return LAMA_OK;
}

// Map::bounds (map.cpp:139-157): the anchors of the allocated patches, max + patch_length on every axis
int OccMap3Dev::bounds(uint32_t mn[3], uint32_t mx[3], int* patches) const
{
    const Impl& d = *d_;
    int n = 0;
    for (int k = 0; k < 3; ++k) { mn[k] = 0xFFFFFFFFu; mx[k] = 0; }
    for (int i = 0; i < d.ndir; ++i) {
        if (d.h_dir[i] < 0) continue;
        uint32_t a[3];
        d.anchor(i, a);
        for (int k = 0; k < 3; ++k) {
            mn[k] = std::min(mn[k], a[k]);
            mx[k] = std::max(mx[k], a[k]);
        }
        ++n;
    }
    for (int k = 0; k < 3; ++k) mx[k] += kPatchLen;
    if (patches) *patches = n;
    return LAMA_OK;
}

int OccMap3Dev::export_box(const uint32_t lo[3], const int32_t size[3], uint32_t* words, uint8_t* known)
{
    Impl& d = *d_;
    if (size[0] < 1 || size[1] < 1 || size[2] < 1) { err_ = "empty box"; return LAMA_ERR_ARG; }
    const size_t n = (size_t)size[0] * size[1] * size[2];
    OM_TRY(cudaSetDevice(d.device));
    OM_TRY(d.ensure(d.qout, n * 4));
    OM_TRY(d.ensure(d.qflag, n));
    k_om3_export<<<std::min<uint64_t>(8192, blocks_for(n)), kThreads, 0, d.stream>>>(d.view(), lo[0], lo[1], lo[2], size[0], size[1], size[2],
                                                                                     (uint32_t*)d.qout.p, (uint8_t*)d.qflag.p);
    OM_TRY(cudaGetLastError());
    if (words) OM_TRY(cudaMemcpyAsync(words, d.qout.p, n * 4, cudaMemcpyDeviceToHost, d.stream));
    if (known) OM_TRY(cudaMemcpyAsync(known, d.qflag.p, n, cudaMemcpyDeviceToHost, d.stream));
    OM_TRY(cudaStreamSynchronize(d.stream));
    return LAMA_OK;
}

// Map::write (map.cpp:490-529) with is_3d: patches in ascending directory index (the reference iterates an unordered_map)
int OccMap3Dev::write(const std::string& path)
{
    Impl& d = *d_;
    OM_TRY(cudaSetDevice(d.device));
    SdmFile f;
    f.header.magic = kSdmMagic;
    f.header.version = kSdmVersion;
    f.header.cell_size = 4;
    f.header.patch_length = kPatchLen;
    f.header.resolution = (float)d.resolution;
    f.header.is_3d = 1;
    std::vector<int> list;
    for (int i = 0; i < d.ndir; ++i)
        if (d.h_dir[i] >= 0) list.push_back(i);
    f.cells.resize(list.size() * (size_t)kOm3Cells * 4);
    f.masks.resize(list.size() * (size_t)kOm3Cells / 64);
    for (size_t j = 0; j < list.size(); ++j) {
        uint32_t a[3];
        d.anchor(list[j], a);
        f.ids.push_back(((uint64_t)(a[0] >> kPatchLog2) * kUniversalConstant + (a[1] >> kPatchLog2)) * kUniversalConstant + (a[2] >> kPatchLog2));   // map.h:153-161
        const int slot = d.h_dir[list[j]];
        OM_TRY(cudaMemcpyAsync(f.cells.data() + j * (size_t)kOm3Cells * 4, d.cells + ((size_t)slot << kOm3Log2Cells), (size_t)kOm3Cells * 4,
                               cudaMemcpyDeviceToHost, d.stream));
        // the mask words are 64-bit (container.cpp:39-43); two little-endian 32-bit known words make one
        OM_TRY(cudaMemcpyAsync(f.masks.data() + j * (size_t)kOm3Cells / 64, d.known + (size_t)slot * kOm3KnownWords, (size_t)kOm3KnownWords * 4,
                               cudaMemcpyDeviceToHost, d.stream));
    }
    OM_TRY(cudaStreamSynchronize(d.stream));
    f.header.num_patches = f.ids.size();
    std::string err;
    if (!sdm_write(path, f, err)) { err_ = err; return LAMA_ERR_ARG; }
    return LAMA_OK;
}

// Map::read (map.cpp:531-575) into an empty map: the cell size and is_3d must match; the file's resolution is taken
int OccMap3Dev::read(const std::string& path)
{
    Impl& d = *d_;
    if (d.used != 0) { err_ = "read needs an empty map"; return LAMA_ERR_STATE; }
    SdmFile f;
    std::string err;
    if (!sdm_read(path, 4, 0, f, err, true)) { err_ = err; return LAMA_ERR_ARG; }
    std::vector<uint32_t> marks((size_t)d.ndir, 0);
    std::vector<int> entry(f.ids.size());
    const uint64_t uc2 = kUniversalConstant * kUniversalConstant;
    for (size_t j = 0; j < f.ids.size(); ++j) {   // Map::p2m (map.h:166-177) with is_3d
        const uint64_t id = f.ids[j];
        const uint64_t px = id / uc2, py = (id % uc2) / kUniversalConstant, pz = id % kUniversalConstant;
        const int di = tsdm_dir_index(d.win, (uint32_t)(px << kPatchLog2), (uint32_t)(py << kPatchLog2), (uint32_t)(pz << kPatchLog2));
        if (di < 0) { err_ = "a patch of " + path + " lies outside the directory window"; return LAMA_ERR_WINDOW; }
        marks[di] = 1;
        entry[j] = di;
    }
    OM_TRY(cudaSetDevice(d.device));
    int rc = d.alloc_marked(marks, err_, d.launches[1]);
    if (rc != LAMA_OK) return rc;
    d.resolution = (double)f.header.resolution;   // map.cpp:548
    d.scale = 1.0 / d.resolution;
    for (size_t j = 0; j < f.ids.size(); ++j) {
        const int slot = d.h_dir[entry[j]];
        OM_TRY(cudaMemcpyAsync(d.cells + ((size_t)slot << kOm3Log2Cells), f.cells.data() + j * (size_t)kOm3Cells * 4, (size_t)kOm3Cells * 4,
                               cudaMemcpyHostToDevice, d.stream));
        OM_TRY(cudaMemcpyAsync(d.known + (size_t)slot * kOm3KnownWords, f.masks.data() + j * (size_t)kOm3Cells / 64, (size_t)kOm3KnownWords * 4,
                               cudaMemcpyHostToDevice, d.stream));
    }
    OM_TRY(cudaStreamSynchronize(d.stream));
    return LAMA_OK;
}

// build_image (export.cpp:46-72): bounds in x / y, the slice z = w2m((0, 0, zed)).z; 90 = no known cell, 255 free, 0 occupied, 127 else
int OccMap3Dev::export_image(double zed, uint8_t* pixels, size_t cap, int dims[2])
{
    Impl& d = *d_;
    uint32_t mn[3], mx[3];
    int np = 0;
    bounds(mn, mx, &np);
    if (np == 0) {
        dims[0] = dims[1] = 0;
        return LAMA_OK;
    }
    const int w = (int)(mx[0] - mn[0]), h = (int)(mx[1] - mn[1]);
    dims[0] = w;
    dims[1] = h;
    if (!pixels || cap < (size_t)w * h) return LAMA_OK;
    const uint32_t lo[3] = {mn[0], mn[1], w2m(zed, d.scale)};
    const int32_t size[3] = {w, h, 1};
    std::vector<uint32_t> words((size_t)w * h);
    std::vector<uint8_t> known((size_t)w * h);
    int rc = export_box(lo, size, words.data(), known.data());
    if (rc != LAMA_OK) return rc;
    for (size_t i = 0; i < words.size(); ++i) {
        if (!known[i]) { pixels[i] = 90; continue; }
        const uint32_t fl = om3_flags(d.kind, true, words[i], d.pp);
        pixels[i] = (fl & 1u) ? 255 : ((fl & 2u) ? 0 : 127);
    }
    return LAMA_OK;
}

}  // namespace lama_b200
