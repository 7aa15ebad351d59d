// patch_store.cuh -- the device patch store of TsdmDev (tsdm.cu), OccMap3Dev (om3d.cu) and DistMap3Dev (ddm3d.cu): one map in a dense
// directory window of patches (patch_window.h) taken from a pool, the map-level plumbing the three share (window setup, cell lookup,
// box exports, z-slice image boxes and the patch placement of .sdm files), and the pipeline that fills a map from a batch of point
// clouds in the reference's order (TsdmDev and OccMap3Dev).
//   1. The map's mark pass checks the window, marks the directory entries it touches and counts every point's records; read_marks
//      reads the status and the marks back.  Nothing in the map is written yet, so a window error leaves it unchanged.
//   2. alloc_marked allocates the marked entries that have no patch, in ascending directory index (a full pool is refused before any
//      write), and k_patch_zero clears them.
//   3. scan_records gives every point its first record, in (cloud, point, step) order, and every cloud its first record.
//   4. for_each_chunk cuts the batch at cloud boundaries into chunks of at most kRecordCap records.
//   5. Per chunk the map emits its records; sort_fold stable-sorts them by cell and k_fold_runs folds each cell's run in record order,
//      loading and storing the cell once.
// Included by tsdm.cu, om3d.cu and ddm3d.cu only: everything here has internal linkage in each.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "cuda_owned.h"
#include "frontend.h"
#include "patch_window.h"
#include "sdm_io.h"

// evaluates a CUDA call; on failure sets err_ to "<call>: <error>" and returns LAMA_ERR_CUDA
#define PS_TRY(...)                                                                                         \
    do {                                                                                                    \
        cudaError_t _e = (__VA_ARGS__);                                                                     \
        if (_e != cudaSuccess) { err_ = std::string(#__VA_ARGS__) + ": " + cudaGetErrorString(_e); return LAMA_ERR_CUDA; } \
    } while (0)

namespace lama_b200 {

int cuda_device_count();   // engine.cu

namespace {

constexpr uint64_t kRecordCap = uint64_t(1) << 24;   // records of one sort chunk (a longer single cloud gets a chunk of its own)
constexpr int kMaxDim = 2048;                         // patches per window axis: window-relative cells fit 16 bits
constexpr int kThreads = 256;
constexpr int32_t kWindow3D[3] = {8, 8, 4};           // the default window of a 3-D map, in patches

inline unsigned blocks_for(uint64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

// A map's device view V has dir (the slot of each directory entry, -1 = absent), the pool's cells and mask (one bit per cell), and
// log2v, the log2 of the cells of a patch: a member, or a static constexpr where it is fixed at compile time.
template <class V>
__device__ __forceinline__ size_t pool_index(const V& v, int slot, uint32_t ci) { return ((size_t)slot << v.log2v) | ci; }

// the pool index of cell (x, y, z) in a store of patches of 1 << log2v cells, or -1 when the cell lies outside the window or its
// patch is absent (the patch lookup of the const get, map.cpp:414-455)
__device__ __forceinline__ int64_t cell_pool_index(const PatchWindow& w, const int32_t* dir, int log2v, uint32_t x, uint32_t y, uint32_t z)
{
    const int di = window_dir_index(w, x, y, z);
    if (di < 0) return -1;
    const int slot = dir[di];
    if (slot < 0) return -1;
    return (int64_t)(((size_t)slot << log2v) | window_cell_index(x, y, z, w.is3d));
}

// the device output planes of a box export
struct Planes { void* p[3]; };

// the box lo + [0, size), x fastest, then y, then z, one grid-stride thread per cell: Cell::put(v, g, i, out) writes entry i of the
// output planes from the cell at pool index g (-1: no cell there)
template <class Cell, class V>
__global__ void k_export_box(V v, PatchWindow w, const int32_t* dir, int log2v, uint32_t x0, uint32_t y0, uint32_t z0, int sx, int sy, int sz, Planes out)
{
    const size_t n = (size_t)sx * sy * sz;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t x = x0 + (uint32_t)(i % sx), y = y0 + (uint32_t)((i / sx) % sy), z = z0 + (uint32_t)(i / ((size_t)sx * sy));
        Cell::put(v, cell_pool_index(w, dir, log2v, x, y, z), i, out);
    }
}

__device__ __forceinline__ int cloud_of(const int64_t* off, int n, int64_t p)
{
    int lo = 0, hi = n;   // the last cloud c with off[c] <= p
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (off[mid] <= p) lo = mid; else hi = mid;
    }
    return lo;
}

template <class V>
__global__ void k_patch_zero(const int32_t* slots, int n, V v)
{
    const size_t per = (size_t)1 << v.log2v, total = per * (size_t)n;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t g = pool_index(v, slots[i >> v.log2v], (uint32_t)(i & (per - 1)));
        v.cells[g] = {};
        if ((g & 31) == 0) v.mask[g >> 5] = 0;
    }
}

__global__ void k_cloud_bounds(const uint64_t* offs, const int64_t* idx, int n, uint64_t* out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = offs[idx[i]];
}

// one thread per run of equal cell keys (directory index << log2v | cell index): Fold::fold(cell, value, args...) of the run's records
// in record order, from the stored cell
template <class Word, class Fold, class V, class... Args>
__global__ void __launch_bounds__(kThreads) k_fold_runs(const Word* __restrict__ keys, const Word* __restrict__ vals, uint64_t n, V v, Args... args)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Word k = keys[i];
    if (i > 0 && keys[i - 1] == k) return;
    const size_t g = pool_index(v, v.dir[k >> v.log2v], (uint32_t)(k & ((1u << v.log2v) - 1)));
    auto cell = v.cells[g];
    for (uint64_t j = i; j < n && keys[j] == k; ++j) Fold::fold(cell, vals[j], args...);
    v.cells[g] = cell;
}

struct PatchStore {
    using Buf = DeviceArray<char>;   // a scratch buffer that grows (Buf::reserve)

    int device = 0;
    Stream stream;
    bool timing = false;
    Event ev[2];
    PatchWindow win{};
    int log2v = 0, ndir = 0, pool = 0, used = 0;
    int end_bit = 0;                // the bits of a record key
    std::vector<int32_t> h_dir;     // the directory, as on the device
    DeviceArray<int32_t> dir_;
    DeviceArray<char> cells_;
    DeviceArray<uint32_t> mask_, status_, marks_;
    int32_t* dir = nullptr;         // the arrays of dir_ .. marks_
    void* cells = nullptr;
    uint32_t* mask = nullptr;
    uint32_t* status = nullptr;
    uint32_t* marks = nullptr;      // per directory entry: touched by this batch
    double ms[3] = {0, 0, 0};
    uint64_t launches[3] = {0, 0, 0};
    Buf pts, off, tf, counts, offs, bound, slots, rk[2], rv[2], temp, box[3];

    PatchStore() = default;
    PatchStore(const PatchStore&) = delete;
    PatchStore& operator=(const PatchStore&) = delete;
    ~PatchStore() { quiesce(); }
    // selects the store's device and waits for its stream: a map's destructor calls it before its own buffers go
    void quiesce() const
    {
        cudaSetDevice(device);
        if (stream) cudaStreamSynchronize(stream);
    }

    // The window of a map's create(): resolution > 0 and patch_size 32; `window` patches per axis (dflt when null; one on z in 2-D),
    // 1..2048 on every axis and at most max_entries in all, centred on center (the origin when null).  LAMA_ERR_ARG when refused.
    static int make_window(double resolution, uint32_t patch_size, const int32_t window[3], const int32_t dflt[3], const double center[3], bool is3d,
                           int64_t max_entries, PatchWindow& w, std::string& err)
    {
        if (!(resolution > 0)) { err = "resolution must be positive"; return LAMA_ERR_ARG; }
        if (patch_size != (uint32_t)kPatchLen) { err = "patch_size must be 32 (the device patch layout)"; return LAMA_ERR_ARG; }
        int32_t dim[3];
        for (int k = 0; k < 3; ++k) dim[k] = window ? window[k] : dflt[k];
        if (!is3d) dim[2] = 1;
        for (int k = 0; k < 3; ++k)
            if (dim[k] < 1 || dim[k] > kMaxDim) { err = "window must be 1..2048 patches per axis"; return LAMA_ERR_ARG; }
        if ((int64_t)dim[0] * dim[1] * dim[2] > max_entries) { err = "window has more than " + std::to_string(max_entries) + " patches"; return LAMA_ERR_ARG; }
        w.is3d = is3d;
        for (int k = 0; k < 3; ++k) {
            w.dim[k] = dim[k];
            const double c = center ? center[k] : 0.0;
            w.base[k] = (k < 2 || is3d) ? (int32_t)(w2m(c, 1.0 / resolution) >> kPatchLog2) - dim[k] / 2 : 0;
        }
        return LAMA_OK;
    }

    // the status of a create() whose CUDA call failed
    static int cuda_failure() { return cuda_device_count() < 1 ? LAMA_ERR_NO_DEVICE : LAMA_ERR_CUDA; }

    // Takes the device and stream of dev (a new non-blocking stream when it names none) and allocates the directory of w, all entries
    // absent, and a pool of dev.pool_slots patches (0: one per entry) of 1 << log2 cells of cell_bytes and one mask bit each.
    // On failure err = "<call>: <error>" of the CUDA call that failed, and the status is cuda_failure().
    int init(const DeviceOptions& dev, const PatchWindow& w, int log2, size_t cell_bytes, std::string& err)
    {
        device = dev.device;
        timing = dev.timing != 0;
        win = w;
        log2v = log2;
        ndir = w.dim[0] * w.dim[1] * w.dim[2];
        pool = dev.pool_slots > 0 ? dev.pool_slots : ndir;
        end_bit = log2v;
        while ((1ll << (end_bit - log2v)) < ndir) ++end_bit;
        h_dir.assign((size_t)ndir, -1);
        const size_t per = (size_t)1 << log2v;
#define PS_INIT(expr)                                                                                        \
        do {                                                                                                 \
            cudaError_t _e = (expr);                                                                         \
            if (_e != cudaSuccess) { err = std::string(#expr) + ": " + cudaGetErrorString(_e); return cuda_failure(); } \
        } while (0)
        PS_INIT(cudaSetDevice(dev.device));
        if (dev.stream)
            stream.borrow(reinterpret_cast<cudaStream_t>(dev.stream));
        else
            PS_INIT(stream.create());
        PS_INIT(ev[0].create(cudaEventDefault));
        PS_INIT(ev[1].create(cudaEventDefault));
        PS_INIT(dir_.alloc((size_t)ndir));
        PS_INIT(marks_.alloc((size_t)ndir));
        PS_INIT(cells_.alloc((size_t)pool * per * cell_bytes));
        PS_INIT(mask_.alloc((size_t)pool * per / 32));
        PS_INIT(status_.alloc(1));
        dir = dir_.get(), marks = marks_.get(), cells = cells_.get(), mask = mask_.get(), status = status_.get();
        PS_INIT(cudaMemcpyAsync(dir, h_dir.data(), (size_t)ndir * 4, cudaMemcpyHostToDevice, stream));
        PS_INIT(cudaStreamSynchronize(stream));
#undef PS_INIT
        return LAMA_OK;
    }

    // ---- timing: kernel_times' ms[k] adds up the time from ev[0] to ev[1]; launches[k] is counted by the map -----------------------
    cudaError_t record(int i) { return timing ? cudaEventRecord(ev[i], stream) : cudaSuccess; }
    // waits for the stream; with timing, adds the time from ev[0] to ev[1] to ms[k]
    cudaError_t finish(int k)
    {
        cudaError_t e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess || !timing) return e;
        float t = 0;
        e = cudaEventElapsedTime(&t, ev[0], ev[1]);
        if (e == cudaSuccess) ms[k] += t;
        return e;
    }
    void kernel_times(double out_ms[3], uint64_t out_launches[3]) const
    {
        for (int k = 0; k < 3; ++k) {
            if (out_ms) out_ms[k] = ms[k];
            if (out_launches) out_launches[k] = launches[k];
        }
    }

    // ---- a batch of point clouds -----------------------------------------------------------------------------------------------------
    // Checks n_clouds clouds, offsets[0] = 0 and non-decreasing (not read without clouds); n_pts = offsets[n_clouds], 0 without clouds
    static int check_clouds(const double* p, const int64_t* offsets, int n_clouds, int64_t& n_pts, std::string& err)
    {
        n_pts = 0;
        if (n_clouds < 0) { err = "negative number of clouds"; return LAMA_ERR_ARG; }
        if (n_clouds == 0) return LAMA_OK;
        if (!offsets || offsets[0] != 0) { err = "offsets must start at 0"; return LAMA_ERR_ARG; }
        for (int k = 0; k < n_clouds; ++k)
            if (offsets[k + 1] < offsets[k]) { err = "offsets must not decrease"; return LAMA_ERR_ARG; }
        n_pts = offsets[n_clouds];
        if (n_pts > 0 && !p) { err = "null points"; return LAMA_ERR_ARG; }
        if (n_pts >= (int64_t)1 << 40) { err = "too many points"; return LAMA_ERR_ARG; }
        return LAMA_OK;
    }

    // Uploads a checked batch: points, offsets and every cloud's Translation(origin) * orientation.  Sizes the per-point record
    // counts and offsets (with one more entry, cleared, past the last point) and the per-cloud bounds, and clears status and marks.
    cudaError_t upload_clouds(const double* p, const int64_t* offsets, int n_clouds, int64_t n_pts, const double* origins, const double* quats)
    {
        std::vector<Affine> h_tf((size_t)n_clouds);
        for (int k = 0; k < n_clouds; ++k) {
            const MovingTf m = moving_tf(origins ? origins + 3 * k : nullptr, quats ? quats + 4 * k : nullptr);
            std::memcpy(h_tf[k].l, m.l, sizeof(m.l));
            std::memcpy(h_tf[k].t, m.t, sizeof(m.t));
        }
        cudaError_t e = pts.reserve((size_t)n_pts * 24);
        if (e == cudaSuccess) e = off.reserve((size_t)(n_clouds + 1) * 8);
        if (e == cudaSuccess) e = tf.reserve((size_t)n_clouds * sizeof(Affine));
        if (e == cudaSuccess) e = counts.reserve((size_t)(n_pts + 1) * 8);
        if (e == cudaSuccess) e = offs.reserve((size_t)(n_pts + 1) * 8);
        if (e == cudaSuccess) e = bound.reserve((size_t)(n_clouds + 1) * 8);
        if (e == cudaSuccess && n_pts) e = cudaMemcpyAsync(pts.get(), p, (size_t)n_pts * 24, cudaMemcpyHostToDevice, stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(off.get(), offsets, (size_t)(n_clouds + 1) * 8, cudaMemcpyHostToDevice, stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(tf.get(), h_tf.data(), (size_t)n_clouds * sizeof(Affine), cudaMemcpyHostToDevice, stream);
        if (e == cudaSuccess) e = cudaMemsetAsync((uint64_t*)counts.get() + n_pts, 0, 8, stream);
        return e == cudaSuccess ? clear_marks() : e;
    }

    cudaError_t clear_marks()
    {
        cudaError_t e = cudaMemsetAsync(status, 0, 4, stream);
        return e == cudaSuccess ? cudaMemsetAsync(marks, 0, (size_t)ndir * 4, stream) : e;
    }

    // after a mark pass: the status word and the marks; waits for the stream
    cudaError_t read_marks(uint32_t& h_status, std::vector<uint32_t>& h_marks)
    {
        h_status = 0;
        h_marks.resize((size_t)ndir);
        cudaError_t e = cudaMemcpyAsync(&h_status, status, 4, cudaMemcpyDeviceToHost, stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(h_marks.data(), marks, (size_t)ndir * 4, cudaMemcpyDeviceToHost, stream);
        return e == cudaSuccess ? cudaStreamSynchronize(stream) : e;
    }

    // allocates the marked entries that have no patch (ascending directory index) and zeroes them; LAMA_ERR_POOL before any change
    template <class V>
    int alloc_marked(const std::vector<uint32_t>& h_marks, const V& v, std::string& err, uint64_t& launch_count)
    {
        std::vector<int32_t> fresh;
        for (int i = 0; i < ndir; ++i)
            if (h_marks[i] && h_dir[i] < 0) fresh.push_back(i);
        if ((int64_t)used + (int64_t)fresh.size() > pool) { err = "the patch pool is exhausted (raise pool_slots)"; return LAMA_ERR_POOL; }
        if (fresh.empty()) return LAMA_OK;
        std::vector<int32_t> sl(fresh.size());
        for (size_t i = 0; i < fresh.size(); ++i) h_dir[fresh[i]] = sl[i] = used++;
        cudaError_t e = slots.reserve(sl.size() * 4);
        if (e == cudaSuccess) e = cudaMemcpyAsync(slots.get(), sl.data(), sl.size() * 4, cudaMemcpyHostToDevice, stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dir, h_dir.data(), (size_t)ndir * 4, cudaMemcpyHostToDevice, stream);
        if (e != cudaSuccess) { err = std::string("patch allocation: ") + cudaGetErrorString(e); return LAMA_ERR_CUDA; }
        k_patch_zero<<<std::min<uint64_t>(4096, blocks_for((uint64_t)sl.size() << log2v)), kThreads, 0, stream>>>((const int32_t*)slots.get(),
                                                                                                              (int)sl.size(), v);
        launch_count += 1;
        return LAMA_OK;
    }

    // exclusive scan of the first n entries of counts into offs
    cudaError_t scan_counts(int64_t n)
    {
        size_t bytes = 0;
        cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const uint64_t*)counts.get(), (uint64_t*)offs.get(), n, stream);
        if (e == cudaSuccess) e = temp.reserve(bytes);
        if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(temp.get(), bytes, (const uint64_t*)counts.get(), (uint64_t*)offs.get(), n, stream);
        return e;
    }

    // offs = every point's first record; h_bound[c] = the first record of cloud c, h_bound[n_clouds] = all records.  Waits for the
    // stream.
    cudaError_t scan_records(int64_t n_pts, int n_clouds, std::vector<uint64_t>& h_bound)
    {
        cudaError_t e = scan_counts(n_pts + 1);
        if (e != cudaSuccess) return e;
        k_cloud_bounds<<<blocks_for(n_clouds + 1), kThreads, 0, stream>>>((const uint64_t*)offs.get(), (const int64_t*)off.get(), n_clouds + 1,
                                                                           (uint64_t*)bound.get());
        h_bound.resize((size_t)n_clouds + 1);
        e = cudaMemcpyAsync(h_bound.data(), bound.get(), h_bound.size() * 8, cudaMemcpyDeviceToHost, stream);
        return e == cudaSuccess ? cudaStreamSynchronize(stream) : e;
    }

    // Cuts clouds [0, n_clouds) at cloud boundaries into chunks of at most kRecordCap records and calls f(c0, c1, records) for each
    // chunk [c0, c1), those without records too; stops at the first result other than LAMA_OK and returns it.
    template <class F>
    static int for_each_chunk(const std::vector<uint64_t>& h_bound, int n_clouds, F&& f)
    {
        for (int c0 = 0; c0 < n_clouds;) {
            int c1 = c0 + 1;
            while (c1 < n_clouds && h_bound[c1 + 1] - h_bound[c0] <= kRecordCap) ++c1;
            const int rc = f(c0, c1, h_bound[c1] - h_bound[c0]);
            if (rc != LAMA_OK) return rc;
            c0 = c1;
        }
        return LAMA_OK;
    }

    // rk[0..1] and rv[0..1] for n records of Word keys and values
    template <class Word>
    cudaError_t ensure_records(uint64_t n)
    {
        cudaError_t e = cudaSuccess;
        for (int b = 0; b < 2 && e == cudaSuccess; ++b) {
            e = rk[b].reserve(n * sizeof(Word));
            if (e == cudaSuccess) e = rv[b].reserve(n * sizeof(Word));
        }
        return e;
    }

    // Stable radix sort of the n records in rk[0] / rv[0] by key (bits 0 .. end_bit) into rk[1] / rv[1]; rk[0] / rv[0] keep the
    // records in record order.  N is CUB's item count type.
    template <class Word, class N>
    cudaError_t sort_records(N n)
    {
        size_t bytes = 0;
        cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const Word*)rk[0].get(), (Word*)rk[1].get(), (const Word*)rv[0].get(), (Word*)rv[1].get(), n, 0,
                                                        end_bit, stream);
        if (e == cudaSuccess) e = temp.reserve(bytes);
        if (e == cudaSuccess)
            e = cub::DeviceRadixSort::SortPairs(temp.get(), bytes, (const Word*)rk[0].get(), (Word*)rk[1].get(), (const Word*)rv[0].get(), (Word*)rv[1].get(), n, 0, end_bit,
                                                stream);
        return e;
    }

    // sort_records, then k_fold_runs over the sorted records
    template <class Word, class Fold, class N, class V, class... Args>
    cudaError_t sort_fold(N n, const V& v, Args... args)
    {
        const cudaError_t e = sort_records<Word>(n);
        if (e != cudaSuccess) return e;
        k_fold_runs<Word, Fold><<<blocks_for((uint64_t)n), kThreads, 0, stream>>>((const Word*)rk[1].get(), (const Word*)rv[1].get(), (uint64_t)n, v, args...);
        return cudaSuccess;
    }

    // ---- the allocated patches -------------------------------------------------------------------------------------------------------
    // Map::bounds (map.cpp:139-157): the anchors of the allocated patches, max + patch_length on every axis
    void bounds(uint32_t mn[3], uint32_t mx[3], int* patches) const
    {
        int n = 0;
        for (int k = 0; k < 3; ++k) { mn[k] = 0xFFFFFFFFu; mx[k] = 0; }
        for (int i = 0; i < ndir; ++i) {
            if (h_dir[i] < 0) continue;
            uint32_t a[3];
            window_anchor(win, i, a);
            for (int k = 0; k < 3; ++k) {
                mn[k] = std::min(mn[k], a[k]);
                mx[k] = std::max(mx[k], a[k]);
            }
            ++n;
        }
        for (int k = 0; k < 3; ++k) mx[k] += kPatchLen;
        if (patches) *patches = n;
    }

    // the directory entries that have a patch, ascending
    std::vector<int32_t> allocated() const
    {
        std::vector<int32_t> list;
        for (int i = 0; i < ndir; ++i)
            if (h_dir[i] >= 0) list.push_back(i);
        return list;
    }

    // ---- exports -----------------------------------------------------------------------------------------------------------------------
    // The box lo + [0, size) through k_export_box<Cell> into Cell::kPlanes planes of Cell::kBytes[k] bytes per cell; each plane k with
    // a non-null host[k] is copied there.  Waits for the stream.
    template <class Cell, class V>
    int export_box(const V& v, const uint32_t lo[3], const int32_t size[3], void* const host[], std::string& err)
    {
        if (size[0] < 1 || size[1] < 1 || size[2] < 1) { err = "empty box"; return LAMA_ERR_ARG; }
        const size_t n = (size_t)size[0] * size[1] * size[2];
        Planes out{};
        cudaError_t e = cudaSetDevice(device);
        for (int k = 0; k < Cell::kPlanes && e == cudaSuccess; ++k) {
            e = box[k].reserve(n * Cell::kBytes[k]);
            out.p[k] = box[k].get();
        }
        if (e == cudaSuccess) {
            k_export_box<Cell><<<std::min<uint64_t>(8192, blocks_for(n)), kThreads, 0, stream>>>(v, win, dir, log2v, lo[0], lo[1], lo[2], size[0], size[1],
                                                                                               size[2], out);
            e = cudaGetLastError();
        }
        for (int k = 0; k < Cell::kPlanes && e == cudaSuccess; ++k)
            if (host[k]) e = cudaMemcpyAsync(host[k], out.p[k], n * Cell::kBytes[k], cudaMemcpyDeviceToHost, stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) { err = std::string("box export: ") + cudaGetErrorString(e); return LAMA_ERR_CUDA; }
        return LAMA_OK;
    }

    // The slice of build_image (export.cpp:46-96) at z = w2m(zed): the x / y bounds of the allocated patches, one cell deep, as lo and
    // size; dims = {width, height}, 0 x 0 without patches.  False when there is no image to export: no patch, or pixels is null or
    // smaller than the image.
    bool image_box(double zed, double scale, const uint8_t* pixels, size_t cap, int dims[2], uint32_t lo[3], int32_t size[3]) const
    {
        uint32_t mn[3], mx[3];
        int np = 0;
        bounds(mn, mx, &np);
        dims[0] = np ? (int)(mx[0] - mn[0]) : 0;
        dims[1] = np ? (int)(mx[1] - mn[1]) : 0;
        lo[0] = mn[0];
        lo[1] = mn[1];
        lo[2] = w2m(zed, scale);
        size[0] = dims[0];
        size[1] = dims[1];
        size[2] = 1;
        return np > 0 && pixels && cap >= (size_t)dims[0] * dims[1];
    }

    // ---- .sdm files ----------------------------------------------------------------------------------------------------------------------
    // Map::write (map.cpp:490-529): the header of a file of cell_size-byte cells and the ids of the allocated patches, in ascending
    // directory index (the reference iterates an unordered_map).  Returns their directory entries, in the same order.
    std::vector<int32_t> sdm_begin(SdmFile& f, uint32_t cell_size, double resolution) const
    {
        sdm_begin_file(f, cell_size, (float)resolution);
        f.header.is_3d = win.is3d ? 1 : 0;
        const std::vector<int32_t> list = allocated();
        for (int32_t i : list) {
            uint32_t a[3];
            window_anchor(win, i, a);
            f.ids.push_back(win.is3d ? m2p(a[0], a[1], a[2]) : m2p(a[0], a[1]));
        }
        f.header.num_patches = list.size();
        return list;
    }

    // Map::read (map.cpp:531-575): entry[j] = the directory entry of the file's patch j (Map::p2m); LAMA_ERR_WINDOW when one lies
    // outside the window
    int sdm_entries(const SdmFile& f, const std::string& path, std::vector<int>& entry, std::string& err) const
    {
        entry.resize(f.ids.size());
        for (size_t j = 0; j < f.ids.size(); ++j) {
            uint32_t a[3] = {0, 0, 0};
            if (win.is3d) p2m(f.ids[j], a[0], a[1], a[2]);
            else p2m(f.ids[j], a[0], a[1]);
            entry[j] = window_dir_index(win, a[0], a[1], a[2]);
            if (entry[j] < 0) { err = "a patch of " + path + " lies outside the directory window"; return LAMA_ERR_WINDOW; }
        }
        return LAMA_OK;
    }

private:
};

}  // namespace

}  // namespace lama_b200
