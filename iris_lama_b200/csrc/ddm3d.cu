// ddm3d.cu -- lama::DynamicDistanceMap with is3d = true on the device: the six-neighbour dynamic brushfire, trilinear distance
// queries, box exports, 3-D .sdm files and z-slice images.
//
// The brushfire.  Parity with the reference needs the exact std::priority_queue pop order (DESIGN.md §12), so update() is one
// sequential thread: k_dm3_brushfire, one CTA of one thread, runs Brushfire3::run (ddm3_core.h) on the device pool.  It first applies
// the queued add / remove ops in list order, then the raise and lower waves.  Both heaps live in global memory, sized by the host.
// Before every op and every pop the kernel checks that the heaps have room for what that step can push; when they do not, it stops
// at that boundary and leaves its progress in Dm3State.  The host then doubles the heap (allocate, copy, free) and launches again.
// A launch also stops after a pop budget (2^20 pops), so no launch runs for long.
//
// Memory safety.  Every cell the brushfire touches lies within R = ceil(l2_max * scale) cells, on every axis, of a cell of an
// admitted batch (or of a read file's obstacle).  The host admits a batch only when each of its cells lies at least R + 1 cells
// inside the window, and only when the directory entries it can reach that have no patch fit in the free pool slots (Dm3Guard).
// The kernel still bounds-checks every address: an out-of-window cell or an exhausted pool gives a scratch cell and an error bit,
// never an unchecked pointer.  Pool offsets are 64-bit (slot << 15, 8-byte cells).
//
// The pool is zeroed once at creation and slots are never freed (the class has no patch deletion), so the brushfire allocates a
// patch with one directory write and one counter increment.
#include "ddm3d.h"
#include "ddm3_core.h"
#include "patch_store.cuh"
#include "sdm_io.h"

#include <cstdlib>

namespace lama_b200 {

namespace {

constexpr uint64_t kPopBudget = uint64_t(1) << 20;     // pops per brushfire launch
constexpr uint32_t kHeapCap0 = 1u << 16;               // initial entries of each heap

struct View {
    int32_t* dir;      // slot of each directory entry, -1 = absent
    uint64_t* cells;   // pool: kDm3Cells words per slot
    uint32_t pool;     // slots
    PatchWindow win;
};

// the Map policy of Brushfire3 on the device pool
struct DevMap3 {
    PatchWindow win;
    int32_t* dir;
    uint64_t* cells;
    uint32_t pool, used, err;
    uint64_t scratch;

    __device__ uint64_t* cell(uint32_t x, uint32_t y, uint32_t z)
    {
        const int di = window_dir_index(win, x, y, z);
        if (di < 0) { err |= kErrWindow; return &scratch; }
        int32_t slot = dir[di];
        if (slot < 0) {
            if (used >= pool) { err |= kErrPoolEmpty; return &scratch; }
            slot = (int32_t)used++;
            dir[di] = slot;
        }
        uint64_t* p = cells + (((size_t)slot << kDm3Log2Cells) | dm3_cell_index(x, y, z));
        if (!(*p & kDm3KnownBit)) *p |= kDm3KnownBit;
        return p;
    }
};

// run(), or with seg_end run_segments() over n_seg segments
__global__ void __launch_bounds__(1) k_dm3_brushfire(View v, uint64_t* rq, uint32_t rcap, uint64_t* lq, uint32_t lcap, const uint32_t* ops,
                                                     uint32_t n_ops, int do_update, uint64_t budget, uint32_t max_sqdist, Dm3State* st,
                                                     const uint32_t* seg_end, uint32_t n_seg, uint32_t* seg_processed)
{
    Dm3State s = *st;
    DevMap3 m{v.win, v.dir, v.cells, v.pool, s.used, 0u, 0ull};
    Brushfire3<DevMap3> b(m, Heap{rq, s.raise_size, rcap}, Heap{lq, s.lower_size, lcap}, max_sqdist);
    if (seg_end) b.run_segments(s, ops, seg_end, n_seg, budget, seg_processed);
    else b.run(s, ops, n_ops, do_update != 0, budget);
    s.raise_size = b.raise_q.size;
    s.lower_size = b.lower_q.size;
    s.used = m.used;
    s.err |= b.err | m.err;
    *st = s;
}

// distance(Vector3ui) (dynamic_distance_map.cpp:140-147) through the const get: an absent or unknown cell, or one without a valid
// obstacle, reads sqrt(max_sqdist) * resolution
__device__ __forceinline__ double dm3_distance_at(const View& v, uint32_t x, uint32_t y, uint32_t z, uint32_t max_sqdist, double resolution)
{
    const int64_t g = cell_pool_index(v.win, v.dir, kDm3Log2Cells, x, y, z);
    uint32_t sq = max_sqdist;
    if (g >= 0) {
        const uint64_t c = v.cells[g];
        if (dm3_known(c) && dm3_valid(c)) sq = dm3_sqdist(c);
    }
    return mul_rn(sqrt((double)sq), resolution);
}

// distance(Vector3d, gradient) (:93-133), one thread per point
__global__ void __launch_bounds__(kThreads) k_dm3_distance(View v, const double* __restrict__ pts, int n, double scale, double resolution,
                                                           uint32_t max_sqdist, double* dist, double* grad)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]}, g[3];
    dist[i] = trilinear_distance(p, scale, [&](uint32_t x, uint32_t y, uint32_t z) { return dm3_distance_at(v, x, y, z, max_sqdist, resolution); }, g);
    if (grad)
        for (int k = 0; k < 3; ++k) grad[3 * i + k] = g[k];
}

__global__ void __launch_bounds__(kThreads) k_dm3_cell_distance(View v, const uint32_t* __restrict__ xyz, int n, double resolution, uint32_t max_sqdist,
                                                                double* dist)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dist[i] = dm3_distance_at(v, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], max_sqdist, resolution);
}

// k_export_box's cell: the word (0 where there is no patch) and its known bit
struct BoxCell {
    static constexpr int kPlanes = 2;
    static constexpr size_t kBytes[kPlanes] = {8, 1};
    static __device__ __forceinline__ void put(const View& v, int64_t g, size_t i, const Planes& out)
    {
        const uint64_t c = g < 0 ? 0ull : v.cells[g];
        ((uint64_t*)out.p[0])[i] = c;
        ((uint8_t*)out.p[1])[i] = dm3_known(c);
    }
};

uint64_t env_u64(const char* name, uint64_t dflt)
{
    const char* s = std::getenv(name);
    if (!s) return dflt;
    const unsigned long long v = std::strtoull(s, nullptr, 10);
    return v > 0 ? (uint64_t)v : dflt;
}

// the smallest r with r * r >= sq
uint32_t reach_of(uint32_t sq)
{
    uint32_t r = 0;
    while ((uint64_t)r * r < sq) ++r;
    return r;
}

}  // namespace

// ---- host side ----------------------------------------------------------------------------------------------------------------
struct DistMap3Dev::Impl : PatchStore {
    double resolution = 0, scale = 0;
    uint32_t max_sqdist = 0;
    Dm3Guard guard;
    Dm3State h_st{};
    DeviceArray<Dm3State> st;
    DeviceArray<uint64_t> heap[2];            // raise, lower
    uint64_t budget = kPopBudget;
    uint64_t runs = 0, grows = 0;
    std::vector<uint32_t> pending;            // queued ops, kDm3OpWords words each
    uint32_t pending_kind[2] = {0, 0};        // queued adds, removes
    Buf ops, qin, qout, qgrad, seg;

    ~Impl() { quiesce(); }
    View view() const { return View{dir, (uint64_t*)cells, (uint32_t)pool, win}; }

    // doubles heap k until it holds `need` entries: allocate, copy the live entries, free
    cudaError_t grow(int k, uint64_t need)
    {
        while (heap[k].size() < need) {
            if (heap[k].size() >= (1u << 30)) return cudaErrorMemoryAllocation;
            DeviceArray<uint64_t> p;
            cudaError_t e = p.alloc(heap[k].size() * 2);
            if (e != cudaSuccess) return e;
            const uint32_t live = k == 0 ? h_st.raise_size : h_st.lower_size;
            if (live) e = cudaMemcpyAsync(p.get(), heap[k].get(), (size_t)live * 8, cudaMemcpyDeviceToDevice, stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
            if (e != cudaSuccess) return e;
            heap[k] = std::move(p);
            ++grows;
        }
        return cudaSuccess;
    }
};

DistMap3Dev* DistMap3Dev::create(double resolution, uint32_t patch_size, double l2_max, const double center[3], const int32_t window[3],
                                 const DeviceOptions& dev, std::string& err, int* code)
{
    PatchWindow win;
    *code = PatchStore::make_window(resolution, patch_size, window, kWindow3D, center, true, kDm3MaxEntries, win, err);
    if (*code != LAMA_OK) return nullptr;
    const double r = std::ceil(l2_max * (1.0 / resolution));
    *code = LAMA_ERR_ARG;
    if (!(r >= 0 && r <= kDmMaxRadius)) { err = "l2_max / resolution exceeds 63 cells (8-bit cell offsets)"; return nullptr; }
    if (dev.pool_slots >= (1 << 24)) { err = "pool_slots must be below 2^24"; return nullptr; }

    DistMap3Dev* t = new DistMap3Dev();
    t->d_ = new Impl();
    Impl& d = *t->d_;
    d.resolution = resolution;
    d.scale = 1.0 / resolution;
    d.max_sqdist = (uint32_t)r * (uint32_t)r;   // setMaxDistance (:149-153)
    d.guard.init(win, (int)r);
    d.budget = env_u64("LAMA_DM3_POP_BUDGET", kPopBudget);                       // test hook: a small pop budget per launch
    const uint64_t cap0 = std::min<uint64_t>(env_u64("LAMA_DM3_HEAP_CAP", kHeapCap0), 1u << 30);   // test hook: a small initial heap
    *code = d.init(dev, win, kDm3Log2Cells, 8, err);
    if (*code != LAMA_OK) { delete t; return nullptr; }
    cudaError_t e = cudaMemsetAsync(d.cells, 0, (size_t)d.pool << kDm3Log2Cells << 3, d.stream);
    if (e == cudaSuccess) e = d.st.alloc(1);
    for (int k = 0; k < 2 && e == cudaSuccess; ++k) e = d.heap[k].alloc(cap0);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d.st.get(), &d.h_st, sizeof(Dm3State), cudaMemcpyHostToDevice, d.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(d.stream);
    if (e != cudaSuccess) {
        err = std::string("DistMap3Dev::create: ") + cudaGetErrorString(e);
        *code = PatchStore::cuda_failure();
        delete t;
        return nullptr;
    }
    return t;
}

DistMap3Dev::~DistMap3Dev() { delete d_; }

uint32_t DistMap3Dev::max_sqdist() const { return d_->max_sqdist; }
double DistMap3Dev::max_distance() const { return std::sqrt((double)d_->max_sqdist) * d_->resolution; }
double DistMap3Dev::resolution() const { return d_->resolution; }
void DistMap3Dev::kernel_times(double ms[3], uint64_t launches[3]) const { d_->kernel_times(ms, launches); }
void DistMap3Dev::run_stats(uint64_t out[4]) const
{
    out[0] = d_->runs;
    out[1] = d_->grows;
    out[2] = d_->heap[0].size();
    out[3] = d_->heap[1].size();
}

int DistMap3Dev::add_remove(const uint32_t* cells_xyz, int n, bool remove)
{
    Impl& d = *d_;
    if (n < 0 || (n > 0 && !cells_xyz)) { err_ = "null argument"; return LAMA_ERR_ARG; }
    if (n == 0) return LAMA_OK;
    if ((uint64_t)d.pending.size() / kDm3OpWords + (uint64_t)n >= (1u << 30)) { err_ = "too many queued ops (call update)"; return LAMA_ERR_ARG; }
    // heap room for every queued op, before anything else changes (growing a heap changes no cell)
    const int k = remove ? 0 : 1;
    PS_TRY(cudaSetDevice(d.device));
    PS_TRY(d.grow(k, (uint64_t)(k == 0 ? d.h_st.raise_size : d.h_st.lower_size) + d.pending_kind[k] + (uint64_t)n + kDm3HeapRoom));
    const int rc = d.guard.admit(cells_xyz, n, 3, d.h_dir, (int64_t)d.pool - (int64_t)d.h_st.used, err_);
    if (rc != 0) return rc == -4 ? LAMA_ERR_WINDOW : LAMA_ERR_POOL;
    const size_t base = d.pending.size();
    d.pending.resize(base + (size_t)kDm3OpWords * n);
    for (int i = 0; i < n; ++i) {
        uint32_t* o = d.pending.data() + base + (size_t)kDm3OpWords * i;
        o[0] = cells_xyz[3 * i];
        o[1] = cells_xyz[3 * i + 1];
        o[2] = cells_xyz[3 * i + 2];
        o[3] = remove ? 1u : 0u;
    }
    d.pending_kind[k] += (uint32_t)n;
    return LAMA_OK;
}

// Launches k_dm3_brushfire until the queued ops are applied and, with do_update, both heaps are empty; grows a heap whenever a launch
// stops for room.  A failed allocation returns LAMA_ERR_CUDA with the map at an op or pop boundary and the rest still queued.
int DistMap3Dev::run(bool do_update, uint32_t* processed)
{
    Impl& d = *d_;
    const uint32_t n_ops = (uint32_t)(d.pending.size() / kDm3OpWords);
    PS_TRY(cudaSetDevice(d.device));
    if (n_ops) {
        PS_TRY(d.ops.reserve(d.pending.size() * 4));
        PS_TRY(cudaMemcpyAsync(d.ops.get(), d.pending.data(), d.pending.size() * 4, cudaMemcpyHostToDevice, d.stream));
    }
    if (do_update) d.h_st.processed = 0;
    const int rc = drive((const uint32_t*)d.ops.get(), n_ops, do_update, nullptr, 0, nullptr);
    if (rc != LAMA_OK) return rc;
    d.pending.clear();
    d.pending_kind[0] = d.pending_kind[1] = 0;
    if (processed) *processed = d.h_st.processed;
    return LAMA_OK;
}

// the launch loop of run() and run_segments() from h_st; on success h_st is back at op 0 and segment 0, and the host directory is
// read back
int DistMap3Dev::drive(const uint32_t* ops, uint32_t n_ops, bool do_update, const uint32_t* seg_end, uint32_t n_seg, uint32_t* seg_processed)
{
    Impl& d = *d_;
    PS_TRY(cudaMemcpyAsync(d.st.get(), &d.h_st, sizeof(Dm3State), cudaMemcpyHostToDevice, d.stream));
    PS_TRY(d.record(0));
    for (;;) {
        k_dm3_brushfire<<<1, 1, 0, d.stream>>>(d.view(), d.heap[0].get(), (uint32_t)d.heap[0].size(), d.heap[1].get(), (uint32_t)d.heap[1].size(), ops, n_ops, do_update ? 1 : 0, d.budget, d.max_sqdist,
                                               d.st.get(), seg_end, n_seg, seg_processed);
        d.launches[0] += 1;
        ++d.runs;
        PS_TRY(cudaGetLastError());
        PS_TRY(cudaMemcpyAsync(&d.h_st, d.st.get(), sizeof(Dm3State), cudaMemcpyDeviceToHost, d.stream));
        PS_TRY(cudaStreamSynchronize(d.stream));
        if (d.h_st.err) {
            err_ = "internal: the brushfire addressed a cell outside the admitted region (error bits " + std::to_string(d.h_st.err) + ")";
            return LAMA_ERR_STATE;
        }
        if (d.h_st.stop == kDm3Done) break;
        if (d.h_st.stop == kDm3NeedRoom) {
            PS_TRY(d.grow(0, (uint64_t)d.h_st.raise_size + kDm3HeapRoom));
            PS_TRY(d.grow(1, (uint64_t)d.h_st.lower_size + kDm3HeapRoom));
        }
    }
    PS_TRY(d.record(1));
    PS_TRY(d.finish(0));
    d.h_st.next_op = 0;
    d.h_st.seg = 0;
    PS_TRY(cudaMemcpyAsync(d.h_dir.data(), d.dir, (size_t)d.ndir * 4, cudaMemcpyDeviceToHost, d.stream));
    PS_TRY(cudaStreamSynchronize(d.stream));
    d.used = (int)d.h_st.used;
    return LAMA_OK;
}

int DistMap3Dev::flush() { return d_->pending.empty() ? LAMA_OK : run(false, nullptr); }

DistMap3Dev::Coupling DistMap3Dev::coupling() const
{
    const Impl& d = *d_;
    return Coupling{d.device, (void*)d.stream, d.resolution, d.win, d.guard.reach, d.dir, (uint64_t*)d.cells};
}

int DistMap3Dev::admit_entries(const std::vector<uint32_t>& marks, std::vector<uint8_t>& next)
{
    Impl& d = *d_;
    return d.guard.admit_entries(marks, d.h_dir, (int64_t)d.pool - (int64_t)d.h_st.used, next, err_) == 0 ? LAMA_OK : LAMA_ERR_POOL;
}

void DistMap3Dev::commit_reachable(std::vector<uint8_t>& next) { d_->guard.reachable.swap(next); }

int DistMap3Dev::alloc_entries(const std::vector<uint32_t>& marks, void* done)
{
    Impl& d = *d_;
    PS_TRY(cudaSetDevice(d.device));
    bool fresh = false;
    for (int i = 0; i < d.ndir; ++i)
        if (marks[(size_t)i] && d.h_dir[(size_t)i] < 0) {
            if (d.h_st.used >= (uint32_t)d.pool) { err_ = "internal: an admitted batch found the pool full"; return LAMA_ERR_STATE; }
            d.h_dir[(size_t)i] = (int32_t)d.h_st.used++;   // the pool was zeroed at creation and slots are never freed
            fresh = true;
        }
    if (fresh) {
        d.used = (int)d.h_st.used;
        PS_TRY(cudaMemcpyAsync(d.dir, d.h_dir.data(), (size_t)d.ndir * 4, cudaMemcpyHostToDevice, d.stream));
        PS_TRY(cudaMemcpyAsync(d.st.get(), &d.h_st, sizeof(Dm3State), cudaMemcpyHostToDevice, d.stream));
    }
    PS_TRY(cudaEventRecord((cudaEvent_t)done, d.stream));
    return LAMA_OK;
}

int DistMap3Dev::run_segments(const uint32_t* ops, const std::vector<uint32_t>& seg_end, uint32_t* processed, void* wait)
{
    Impl& d = *d_;
    const uint32_t n_seg = (uint32_t)seg_end.size();
    if (n_seg == 0) return LAMA_OK;
    PS_TRY(cudaSetDevice(d.device));
    if (wait) PS_TRY(cudaStreamWaitEvent(d.stream, (cudaEvent_t)wait, 0));
    PS_TRY(d.seg.reserve((size_t)n_seg * 8));
    uint32_t* dseg = (uint32_t*)d.seg.get();
    PS_TRY(cudaMemcpyAsync(dseg, seg_end.data(), (size_t)n_seg * 4, cudaMemcpyHostToDevice, d.stream));
    d.h_st.processed = 0;
    d.h_st.seg = 0;
    const int rc = drive(ops, seg_end.back(), true, dseg, n_seg, dseg + n_seg);
    if (rc != LAMA_OK) return rc;
    PS_TRY(cudaMemcpyAsync(processed, dseg + n_seg, (size_t)n_seg * 4, cudaMemcpyDeviceToHost, d.stream));
    PS_TRY(cudaStreamSynchronize(d.stream));
    d.h_st.processed = 0;
    return LAMA_OK;
}

int DistMap3Dev::update(uint32_t* processed)
{
    if (processed) *processed = 0;
    return run(true, processed);
}

int DistMap3Dev::distance(const double* pts_xyz, int n, double* dist, double* gradient)
{
    Impl& d = *d_;
    if (n < 0 || (n > 0 && (!pts_xyz || !dist))) { err_ = "null argument"; return LAMA_ERR_ARG; }
    if (n == 0) return LAMA_OK;
    int rc = flush();
    if (rc != LAMA_OK) return rc;
    PS_TRY(cudaSetDevice(d.device));
    PS_TRY(d.qin.reserve((size_t)n * 24));
    PS_TRY(d.qout.reserve((size_t)n * 8));
    if (gradient) PS_TRY(d.qgrad.reserve((size_t)n * 24));
    PS_TRY(cudaMemcpyAsync(d.qin.get(), pts_xyz, (size_t)n * 24, cudaMemcpyHostToDevice, d.stream));
    PS_TRY(d.record(0));
    k_dm3_distance<<<blocks_for(n), kThreads, 0, d.stream>>>(d.view(), (const double*)d.qin.get(), n, d.scale, d.resolution, d.max_sqdist, (double*)d.qout.get(),
                                                             gradient ? (double*)d.qgrad.get() : nullptr);
    d.launches[1] += 1;
    PS_TRY(cudaGetLastError());
    PS_TRY(d.record(1));
    PS_TRY(cudaMemcpyAsync(dist, d.qout.get(), (size_t)n * 8, cudaMemcpyDeviceToHost, d.stream));
    if (gradient) PS_TRY(cudaMemcpyAsync(gradient, d.qgrad.get(), (size_t)n * 24, cudaMemcpyDeviceToHost, d.stream));
    PS_TRY(d.finish(1));
    return LAMA_OK;
}

int DistMap3Dev::cell_distance(const uint32_t* cells_xyz, int n, double* dist)
{
    Impl& d = *d_;
    if (n < 0 || (n > 0 && (!cells_xyz || !dist))) { err_ = "null argument"; return LAMA_ERR_ARG; }
    if (n == 0) return LAMA_OK;
    int rc = flush();
    if (rc != LAMA_OK) return rc;
    PS_TRY(cudaSetDevice(d.device));
    PS_TRY(d.qin.reserve((size_t)n * 12));
    PS_TRY(d.qout.reserve((size_t)n * 8));
    PS_TRY(cudaMemcpyAsync(d.qin.get(), cells_xyz, (size_t)n * 12, cudaMemcpyHostToDevice, d.stream));
    PS_TRY(d.record(0));
    k_dm3_cell_distance<<<blocks_for(n), kThreads, 0, d.stream>>>(d.view(), (const uint32_t*)d.qin.get(), n, d.resolution, d.max_sqdist, (double*)d.qout.get());
    d.launches[2] += 1;
    PS_TRY(cudaGetLastError());
    PS_TRY(d.record(1));
    PS_TRY(cudaMemcpyAsync(dist, d.qout.get(), (size_t)n * 8, cudaMemcpyDeviceToHost, d.stream));
    PS_TRY(d.finish(2));
    return LAMA_OK;
}

int DistMap3Dev::bounds(uint32_t mn[3], uint32_t mx[3], int* patches)
{
    const int rc = flush();
    if (rc != LAMA_OK) return rc;
    d_->PatchStore::bounds(mn, mx, patches);
    return LAMA_OK;
}

int DistMap3Dev::export_box(const uint32_t lo[3], const int32_t size[3], uint64_t* words, uint8_t* known)
{
    int rc = flush();
    if (rc != LAMA_OK) return rc;
    void* const host[] = {words, known};
    rc = d_->export_box<BoxCell>(d_->view(), lo, size, host, err_);
    if (rc == LAMA_OK) d_->launches[2] += 1;
    return rc;
}

// Map::write (map.cpp:490-529) with is_3d and writeParameters (:200-203): 10-byte distance_t cells, patches in ascending directory
// index (the reference iterates an unordered_map)
int DistMap3Dev::write(const std::string& path)
{
    Impl& d = *d_;
    int rc = flush();
    if (rc != LAMA_OK) return rc;
    PS_TRY(cudaSetDevice(d.device));
    SdmFile f;
    const std::vector<int32_t> list = d.sdm_begin(f, sizeof(SdmDistanceCell), d.resolution);
    f.params.resize(4);
    std::memcpy(f.params.data(), &d.max_sqdist, 4);
    f.cells.assign(list.size() * (size_t)kDm3Cells * sizeof(SdmDistanceCell), 0);
    f.masks.assign(list.size() * (size_t)kDm3Cells / 64, 0);
    std::vector<uint64_t> words((size_t)kDm3Cells);
    const View v = d.view();
    for (size_t j = 0; j < list.size(); ++j) {
        PS_TRY(cudaMemcpyAsync(words.data(), v.cells + ((size_t)d.h_dir[list[j]] << kDm3Log2Cells), (size_t)kDm3Cells * 8, cudaMemcpyDeviceToHost, d.stream));
        PS_TRY(cudaStreamSynchronize(d.stream));
        SdmDistanceCell* c = reinterpret_cast<SdmDistanceCell*>(f.cells.data()) + j * (size_t)kDm3Cells;
        uint64_t* mask = f.masks.data() + j * (size_t)kDm3Cells / 64;
        for (int i = 0; i < kDm3Cells; ++i) {
            const uint64_t w = words[(size_t)i];
            if (!dm3_known(w)) continue;   // never written: the calloc'd zeros of Container::alloc (container.cpp:78-95)
            mask[i >> 6] |= uint64_t(1) << (i & 63);
            for (int k = 0; k < 3; ++k) c[i].obstacle[k] = (int16_t)dm3_off(w, k);
            c[i].sqdist = (uint16_t)dm3_sqdist(w);
            c[i].valid_obstacle = dm3_valid(w);
            c[i].is_queued = dm3_queued(w);
        }
    }
    std::string err;
    if (!sdm_write(path, f, err)) { err_ = err; return LAMA_ERR_ARG; }
    return LAMA_OK;
}

// Map::read (map.cpp:531-575) and readParameters (:205-208) into an empty map: the file's resolution and max_sqdist are taken.  The
// whole file is checked before anything changes: every patch inside the window (LAMA_ERR_WINDOW), the invariants every state the
// API makes keeps (an unknown cell is all zero, a valid cell has sqdist = |offset|^2 < max_sqdist, an invalid one sqdist 0 and offset
// 0; LAMA_ERR_ARG), a reach of at most 63 cells (LAMA_ERR_ARG), every valid cell's obstacle at least reach + 1 cells inside the window
// (LAMA_ERR_WINDOW), and the patches plus those the brushfire could reach from the file's obstacles within the pool (LAMA_ERR_POOL).
int DistMap3Dev::read(const std::string& path)
{
    Impl& d = *d_;
    if (d.h_st.used != 0 || !d.pending.empty() || d.h_st.raise_size || d.h_st.lower_size) { err_ = "read needs an empty map"; return LAMA_ERR_STATE; }
    SdmFile f;
    std::string err;
    if (!sdm_read(path, sizeof(SdmDistanceCell), 4, f, err, true)) { err_ = err; return LAMA_ERR_ARG; }
    uint32_t msq = 0;
    std::memcpy(&msq, f.params.data(), 4);
    const uint32_t R = reach_of(msq);
    if (R > (uint32_t)kDmMaxRadius) { err_ = "the file's max_sqdist " + std::to_string(msq) + " is a reach above 63 cells"; return LAMA_ERR_ARG; }
    if (!(f.header.resolution > 0)) { err_ = "the file's resolution is not positive"; return LAMA_ERR_ARG; }
    std::vector<int> entry;
    const int rc = d.sdm_entries(f, path, entry, err_);
    if (rc != LAMA_OK) return rc;
    std::vector<int32_t> file_dir((size_t)d.ndir, -1);
    for (size_t j = 0; j < f.ids.size(); ++j) {
        if (file_dir[(size_t)entry[j]] >= 0) { err_ = path + " holds a patch twice"; return LAMA_ERR_ARG; }
        file_dir[(size_t)entry[j]] = (int32_t)j;
    }
    if ((int64_t)f.ids.size() > d.pool) { err_ = "the file has more patches than the pool has slots (raise pool_slots)"; return LAMA_ERR_POOL; }
    Dm3Guard guard;
    guard.init(d.win, (int)R);
    std::vector<uint64_t> words(f.ids.size() * (size_t)kDm3Cells, 0);
    const SdmDistanceCell* cells = reinterpret_cast<const SdmDistanceCell*>(f.cells.data());
    for (size_t j = 0; j < f.ids.size(); ++j) {
        uint32_t a[3];
        window_anchor(d.win, entry[j], a);
        for (int i = 0; i < kDm3Cells; ++i) {
            const SdmDistanceCell& c = cells[j * (size_t)kDm3Cells + i];
            const bool known = (f.masks[j * (size_t)kDm3Cells / 64 + (i >> 6)] >> (i & 63)) & 1u;
            const int o[3] = {c.obstacle[0], c.obstacle[1], c.obstacle[2]};
            const int64_t sq = (int64_t)o[0] * o[0] + (int64_t)o[1] * o[1] + (int64_t)o[2] * o[2];
            const bool bad_flags = c.valid_obstacle > 1 || c.is_queued > 1;
            if (!known) {
                if (o[0] || o[1] || o[2] || c.sqdist || c.valid_obstacle || c.is_queued) { err_ = path + ": an unknown cell is not zero"; return LAMA_ERR_ARG; }
                continue;
            }
            if (bad_flags || (c.valid_obstacle ? (sq != c.sqdist || c.sqdist >= msq) : (sq != 0 || c.sqdist != 0))) {
                err_ = path + ": a cell breaks the distance map invariants (valid: sqdist = |offset|^2 < max_sqdist; invalid: all zero)";
                return LAMA_ERR_ARG;
            }
            const uint32_t x = a[0] | (i & 31), y = a[1] | ((i >> 5) & 31), z = a[2] | (i >> 10);
            if (c.valid_obstacle) {
                const uint32_t ob[3] = {x + (uint32_t)o[0], y + (uint32_t)o[1], z + (uint32_t)o[2]};
                if (!guard.inside(ob[0], ob[1], ob[2])) { err_ = path + ": an obstacle lies less than reach + 1 cells inside the window"; return LAMA_ERR_WINDOW; }
                guard.mark(guard.reachable, ob[0], ob[1], ob[2]);
            }
            words[j * (size_t)kDm3Cells + i] = dm3_pack(c.sqdist, o[0], o[1], o[2], c.valid_obstacle, c.is_queued);
        }
    }
    if ((int64_t)f.ids.size() + Dm3Guard::missing(guard.reachable, file_dir) > d.pool) {
        err_ = "the patches the file's obstacles can reach exceed the pool (raise pool_slots)";
        return LAMA_ERR_POOL;
    }
    // commit: slots in file order
    PS_TRY(cudaSetDevice(d.device));
    std::vector<int32_t> h_dir((size_t)d.ndir, -1);
    for (size_t j = 0; j < f.ids.size(); ++j) {
        h_dir[(size_t)entry[j]] = (int32_t)j;
        PS_TRY(cudaMemcpyAsync((uint64_t*)d.cells + (j << kDm3Log2Cells), words.data() + j * (size_t)kDm3Cells, (size_t)kDm3Cells * 8, cudaMemcpyHostToDevice,
                               d.stream));
    }
    Dm3State s{};
    s.used = (uint32_t)f.ids.size();
    PS_TRY(cudaMemcpyAsync(d.dir, h_dir.data(), (size_t)d.ndir * 4, cudaMemcpyHostToDevice, d.stream));
    PS_TRY(cudaMemcpyAsync(d.st.get(), &s, sizeof(Dm3State), cudaMemcpyHostToDevice, d.stream));
    PS_TRY(cudaStreamSynchronize(d.stream));
    d.h_dir = h_dir;
    d.h_st = s;
    d.used = (int)s.used;
    d.resolution = (double)f.header.resolution;   // map.cpp:548
    d.scale = 1.0 / d.resolution;
    d.max_sqdist = msq;                           // :205-208
    d.guard = guard;
    return LAMA_OK;
}

// build_image (export.cpp:74-96) of the z-slice at w2m((0, 0, zed)).z, through the 2-D pixel rule of sdm_io.h
int DistMap3Dev::export_image(double zed, uint8_t* pixels, size_t cap, int dims[2])
{
    Impl& d = *d_;
    int rc = flush();
    if (rc != LAMA_OK) return rc;
    uint32_t lo[3];
    int32_t size[3];
    if (!d.image_box(zed, d.scale, pixels, cap, dims, lo, size)) return LAMA_OK;
    const size_t n = (size_t)size[0] * size[1];
    std::vector<uint64_t> words(n);
    std::vector<uint8_t> known(n);
    rc = export_box(lo, size, words.data(), known.data());
    if (rc != LAMA_OK) return rc;
    std::vector<uint16_t> sqdist(n);
    std::vector<uint8_t> valid(n);
    for (size_t i = 0; i < n; ++i) {
        sqdist[i] = (uint16_t)dm3_sqdist(words[i]);
        valid[i] = dm3_valid(words[i]);
    }
    sdm_distance_image(SdmWindow{lo[0], lo[1], size[0], size[1]}, sqdist.data(), valid.data(), known.data(), d.max_sqdist, d.resolution, pixels);
    return LAMA_OK;
}

}  // namespace lama_b200
