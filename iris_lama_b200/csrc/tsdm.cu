// tsdm.cu -- lama::TruncatedSignedDistanceMap on the device (src/sdm/truncated_signed_distance_map.cpp): ordered fusion of
// point clouds, distance queries, exports and marching cubes.
//
// Fusion.  The reference folds every walked voxel into a float running average, so the result depends on the order of the
// updates.  insert_point_clouds keeps that order without serialising the walk, in the manner of the ray cast's candidate replay
// (ray_core.h): every update is logged as a record and each cell's records are replayed in the reference's order.
//   1. k_tsdm_hash: per point, the hit and its 3-D key; a per-cloud hash on (cloud, key) with atomicMin of the point index keeps
//      the first point of every key, as insertPointCloud's KeySet does.
//   2. k_tsdm_walk<false>: every surviving point walks its ray, checks the window, marks the directory entries it touches and
//      counts its records (voxels that are not skipped).  Nothing in the map is written yet: a window error leaves it unchanged.
//   3. The host allocates the marked patches (ascending directory index) from the pool; k_tsdm_zero clears them.
//   4. An exclusive scan of the counts gives every point its first record, in (cloud, point, step) order.  The batch is cut at
//      cloud boundaries into chunks of at most kRecordCap records; per chunk k_tsdm_walk<true> sets the "on" bits of every walked
//      voxel (skipped ones too, as the reference's mutable get() does) and writes the records, a stable radix sort orders them by
//      cell, and k_tsdm_fold folds each run of equal keys in record order, loading and storing its cell once.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "mc_table.h"
#include "tsdm.h"
#include "tsdm_core.h"

namespace lama_b200 {

namespace {

constexpr int64_t kHashPoints = 1 << 20;               // points of one dedupe pass (the hash has >= 2x as many slots)
constexpr int kHashClouds = 65535;                      // clouds of one dedupe pass (16 bits of the hash key)
constexpr uint64_t kRecordCap = uint64_t(1) << 24;      // records of one sort chunk (a longer single cloud gets a chunk of its own)
constexpr int kMaxDim = 2048;                           // patches per window axis: window-relative cells fit 16 bits
constexpr int kThreads = 256;

__constant__ int8_t c_mc_tri[256][kMcRow];
__constant__ uint8_t c_mc_ntri[256];

struct View {
    const int32_t* dir;   // slot of each directory entry, -1 = absent
    float2* cells;        // pool: {distance, weight} per cell
    uint32_t* on;         // pool: one bit per cell
    TsdmWindow w;
    int log2v;            // log2 of the cells of a patch: 10 (2-D) or 15 (3-D)
};

__device__ __forceinline__ size_t pool_index(const View& v, int slot, uint32_t ci) { return ((size_t)slot << v.log2v) | ci; }

// the const get() (map.cpp:414-455): false when the patch is absent or the cell is off
__device__ __forceinline__ bool cell_get(const View& v, uint32_t x, uint32_t y, uint32_t z, float2& out)
{
    const int di = tsdm_dir_index(v.w, x, y, z);
    if (di < 0) return false;
    const int slot = v.dir[di];
    if (slot < 0) return false;
    const size_t g = pool_index(v, slot, tsdm_cell_index(x, y, z, v.w.is3d));
    if (!((v.on[g >> 5] >> (g & 31)) & 1u)) return false;
    out = v.cells[g];
    return true;
}

struct FuseParams {
    const double* pts;
    const int64_t* offsets;   // n_clouds + 1
    const Affine* tf;         // per cloud: Translation(sensor_origin_) * sensor_orientation_
    int n_clouds;
    int64_t p0, p1;           // the points of this pass
    int c0;                   // first cloud of this pass
    TsdmParams prm;
    uint64_t* hkeys;
    uint32_t* hval;
    uint32_t hmask;
    uint32_t* hslot;          // per point of the pass: its hash slot, ~0 when the hit is outside the window
    uint8_t* surv;            // per point: first of its key in its cloud
    uint64_t* counts;         // per point: records
    const uint64_t* offs;     // exclusive scan of counts
    uint64_t rec_base;
    uint64_t* rkeys;          // record: (directory index << log2v) | cell index
    uint64_t* rvals;          // record: distance bits | weight bits << 32
    uint32_t* marks;          // per directory entry: touched by this batch
    uint32_t* inserted;       // per cloud: distinct hit keys
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

__device__ __forceinline__ void point_hit(const FuseParams& f, int64_t p, int c, double hit[3])
{
    apply_tf(f.tf[c], f.pts[3 * p], f.pts[3 * p + 1], f.pts[3 * p + 2], hit);
}

__device__ __forceinline__ uint32_t hash_slot(uint64_t k, uint32_t mask)
{
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (uint32_t)k & mask;
}

// insertPointCloud's KeySet (:146-153): slot of (cloud, w2m(hit)); the smallest point index of each key survives
__global__ void __launch_bounds__(kThreads) k_tsdm_hash(FuseParams f, View v)
{
    const int64_t p = f.p0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= f.p1) return;
    const int c = cloud_of(f.offsets, f.n_clouds, p);
    double hit[3];
    point_hit(f, p, c, hit);
    uint32_t k[3];
    for (int i = 0; i < 3; ++i) k[i] = w2m(hit[i], f.prm.scale);
    const TsdmWindow& w = v.w;
    const uint32_t rx = k[0] - ((uint32_t)w.base[0] << kPatchLog2), ry = k[1] - ((uint32_t)w.base[1] << kPatchLog2);
    // 2-D: z is not addressed, but it is part of the key; it must lie within 2^15 cells of world z = 0
    const uint32_t rz = w.is3d ? k[2] - ((uint32_t)w.base[2] << kPatchLog2) : k[2] - kMapOffsetCells + 32768u;
    if (rx >= ((uint32_t)w.dim[0] << kPatchLog2) || ry >= ((uint32_t)w.dim[1] << kPatchLog2) ||
        rz >= (w.is3d ? (uint32_t)w.dim[2] << kPatchLog2 : 65536u)) {
        atomicOr(f.status, kErrWindow);
        f.hslot[p - f.p0] = ~0u;
        return;
    }
    const uint64_t key = ((uint64_t)(c - f.c0) << 48) | ((uint64_t)rz << 32) | ((uint64_t)ry << 16) | rx;
    uint32_t s = hash_slot(key, f.hmask);
    for (;;) {
        const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(&f.hkeys[s]), ~0ull, (unsigned long long)key);
        if (prev == ~0ull || prev == key) break;
        s = (s + 1) & f.hmask;
    }
    atomicMin(&f.hval[s], (uint32_t)(p - f.p0));
    f.hslot[p - f.p0] = s;
}

// kEmit = false: survivors, window check, directory marks and record counts.  kEmit = true: "on" bits and records.
template <bool kEmit>
__global__ void __launch_bounds__(kThreads) k_tsdm_walk(FuseParams f, View v)
{
    const int64_t p = f.p0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= f.p1) return;
    const int c = cloud_of(f.offsets, f.n_clouds, p);
    if (!kEmit) {
        const uint32_t s = f.hslot[p - f.p0];
        const bool first = s != ~0u && f.hval[s] == (uint32_t)(p - f.p0);
        f.surv[p] = first;
        f.counts[p] = 0;
        if (!first) return;
        atomicAdd(&f.inserted[c], 1u);
    } else if (!f.surv[p]) {
        return;
    }
    double hit[3];
    point_hit(f, p, c, hit);
    const TsdmRay r = tsdm_ray(f.tf[c].t, hit, f.prm);
    RayWalk3 w(r.cells);
    uint64_t n = 0, out = kEmit ? f.offs[p] - f.rec_base : 0;
    while (w.next()) {
        const int di = tsdm_dir_index(v.w, w.x, w.y, w.z);
        if (!kEmit) {
            if (di < 0) {
                atomicOr(f.status, kErrWindow);
                return;
            }
            if (!f.marks[di]) f.marks[di] = 1;
        }
        float d, wt;
        const bool keep = tsdm_sample(r, w.x, w.y, w.z, f.prm, d, wt);
        if (kEmit) {
            const uint32_t ci = tsdm_cell_index(w.x, w.y, w.z, v.w.is3d);
            const size_t g = pool_index(v, v.dir[di], ci);
            atomicOr(&v.on[g >> 5], 1u << (g & 31));
            if (keep) {
                f.rkeys[out] = ((uint64_t)di << v.log2v) | ci;
                f.rvals[out] = (uint64_t)__float_as_uint(d) | ((uint64_t)__float_as_uint(wt) << 32);
                ++out;
            }
        } else {
            n += keep;
        }
    }
    if (!kEmit) f.counts[p] = n;
}

__global__ void k_tsdm_zero(const int32_t* slots, int n, View v)
{
    const size_t per = (size_t)1 << v.log2v, total = per * (size_t)n;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t g = pool_index(v, slots[i >> v.log2v], (uint32_t)(i & (per - 1)));
        v.cells[g] = make_float2(0.f, 0.f);
        if ((g & 31) == 0) v.on[g >> 5] = 0;
    }
}

__global__ void k_tsdm_gather(const uint64_t* offs, const int64_t* idx, int n, uint64_t* out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = offs[idx[i]];
}

// one thread per run of equal cell keys: the run's records in (cloud, point, step) order, from the stored cell
__global__ void __launch_bounds__(kThreads) k_tsdm_fold(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ vals, uint64_t n, View v,
                                                         float max_weight)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t k = keys[i];
    if (i > 0 && keys[i - 1] == k) return;
    const size_t g = pool_index(v, v.dir[k >> v.log2v], (uint32_t)(k & ((1u << v.log2v) - 1)));
    float2 cell = v.cells[g];
    for (uint64_t j = i; j < n && keys[j] == k; ++j) {
        const uint64_t r = vals[j];
        tsdm_fold(cell.x, cell.y, __uint_as_float((uint32_t)r), __uint_as_float((uint32_t)(r >> 32)), max_weight);
    }
    v.cells[g] = cell;
}

// distance(Vector3d, gradient) (:59-130) of n points
__global__ void __launch_bounds__(kThreads) k_tsdm_distance(const double* __restrict__ pts, int n, View v, TsdmParams prm, double* dist, double* grad)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    auto value = [&](uint32_t x, uint32_t y, uint32_t z) -> double {   // distance(Vector3ui), :132-139
        float2 c;
        if (!cell_get(v, x, y, z, c) || c.y == 0.0f) return (double)prm.truncate;
        return (double)c.x;
    };
    double g[3];
    dist[i] = tsdm_distance(&pts[3 * i], prm, value, g);
    for (int k = 0; k < 3; ++k) grad[3 * i + k] = g[k];
}

__global__ void k_tsdm_export(View v, uint32_t x0, uint32_t y0, uint32_t z0, int w, int h, int dd, float* dist, float* weight, uint8_t* on)
{
    const size_t n = (size_t)w * h * dd;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t x = x0 + (uint32_t)(i % w), y = y0 + (uint32_t)((i / w) % h), z = z0 + (uint32_t)(i / ((size_t)w * h));
        float2 c = make_float2(0.f, 0.f);
        const bool b = cell_get(v, x, y, z, c);
        dist[i] = c.x;
        weight[i] = c.y;
        on[i] = b;
    }
}

// toMesh (:220-272): one thread per cell of the listed patches (ascending directory index, then cell index).  kEmit = false: the
// vertex count of the cell; true: its vertices from offs.
template <bool kEmit>
__global__ void __launch_bounds__(kThreads) k_tsdm_mesh(const int32_t* __restrict__ list, int n_list, View v, double scale, uint64_t* counts,
                                                         const uint64_t* offs, float* out)
{
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ((uint64_t)n_list << v.log2v)) return;
    const int di = list[t >> v.log2v];
    const uint32_t ci = (uint32_t)(t & ((1u << v.log2v) - 1));
    const size_t g = pool_index(v, v.dir[di], ci);
    int config = -1;
    float pos[8][3], sdf[8];
    if ((v.on[g >> 5] >> (g & 31)) & 1u) {   // visit_all_cells: every "on" cell, at p2m(patch) + c2m(cell)
        const int px = di % v.w.dim[0], py = (di / v.w.dim[0]) % v.w.dim[1], pz = di / (v.w.dim[0] * v.w.dim[1]);
        const uint32_t x = ((uint32_t)(v.w.base[0] + px) << kPatchLog2) + (ci & (kPatchLen - 1));
        const uint32_t y = ((uint32_t)(v.w.base[1] + py) << kPatchLog2) + ((ci >> kPatchLog2) & (kPatchLen - 1));
        const uint32_t z = v.w.is3d ? ((uint32_t)(v.w.base[2] + pz) << kPatchLog2) + (ci >> (2 * kPatchLog2)) : 0u;
        auto cell = [&](uint32_t a, uint32_t b, uint32_t c, float& s) {
            float2 cc;
            if (!cell_get(v, a, b, c, cc) || cc.y == 0.0f) return false;
            s = cc.x;
            return true;
        };
        config = mc_cube(x, y, z, scale, cell, pos, sdf);
    }
    const int nv = config < 0 ? 0 : 3 * c_mc_ntri[config];
    if (!kEmit) {
        counts[t] = (uint64_t)nv;
        return;
    }
    float* o = out + 3 * offs[t];
    for (int j = 0; j < nv; ++j) mc_edge_vertex(c_mc_tri[config][j], pos, sdf, o + 3 * j);
}

inline unsigned blocks_for(uint64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

}  // namespace

// ---- host side ----------------------------------------------------------------------------------------------------------------
struct TsdmDev::Impl {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false, timing = false;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    double resolution = 0;
    TsdmParams prm{};
    TsdmWindow win{};
    int log2v = 0, ndir = 0, pool = 0, used = 0;
    std::vector<int32_t> h_dir;
    int32_t* dir = nullptr;
    float2* cells = nullptr;
    uint32_t* on = nullptr;
    uint32_t* status = nullptr;
    uint32_t* marks = nullptr;
    double ms[3] = {0, 0, 0};
    uint64_t launches[3] = {0, 0, 0};
    struct Buf { void* p = nullptr; size_t bytes = 0; };
    Buf pts, off, tf, hkeys, hval, hslot, surv, counts, offs, inserted, bound, slots, rk[2], rv[2], temp, qout, list, mesh, box[3];

    View view() const { return View{dir, cells, on, win, log2v}; }
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
        Buf* all[] = {&pts, &off, &tf, &hkeys, &hval, &hslot, &surv, &counts, &offs, &inserted, &bound, &slots, &rk[0], &rk[1], &rv[0], &rv[1],
                      &temp, &qout, &list, &mesh, &box[0], &box[1], &box[2]};
        for (Buf* b : all)
            if (b->p) cudaFree(b->p);
        for (void* p : {(void*)dir, (void*)cells, (void*)on, (void*)status, (void*)marks})
            if (p) cudaFree(p);
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
        if (own_stream && stream) cudaStreamDestroy(stream);
    }
};

#define TS_TRY(expr)                                                                                        \
    do {                                                                                                    \
        cudaError_t _e = (expr);                                                                            \
        if (_e != cudaSuccess) { err_ = std::string(#expr) + ": " + cudaGetErrorString(_e); return LAMA_ERR_CUDA; } \
    } while (0)

TsdmDev* TsdmDev::create(double resolution, uint32_t patch_size, bool is3d, const double center[3], const int32_t window[3], const DeviceOptions& dev,
                         std::string& err)
{
    if (!(resolution > 0)) { err = "resolution must be positive"; return nullptr; }
    if (patch_size != (uint32_t)kPatchLen) { err = "patch_size must be 32 (the device patch layout)"; return nullptr; }
    int32_t dim[3] = {dev.dir_dim, dev.dir_dim, 1};
    if (is3d) { dim[0] = 8; dim[1] = 8; dim[2] = 4; }
    if (window) for (int k = 0; k < 3; ++k) dim[k] = window[k];
    if (!is3d) dim[2] = 1;
    for (int k = 0; k < 3; ++k)
        if (dim[k] < 1 || dim[k] > kMaxDim) { err = "window must be 1..2048 patches per axis"; return nullptr; }
    const int64_t ndir = (int64_t)dim[0] * dim[1] * dim[2];
    if (ndir > (1 << 22)) { err = "window has more than 2^22 patches"; return nullptr; }
    const int pool = dev.pool_slots > 0 ? dev.pool_slots : (int)ndir;

    TsdmDev* t = new TsdmDev();
    t->d_ = new Impl();
    Impl& d = *t->d_;
    d.device = dev.device;
    d.timing = dev.timing != 0;
    d.resolution = resolution;
    d.prm.scale = 1.0 / resolution;
    d.prm.truncate = 0.15f;
    d.prm.delta = (float)(4 * resolution);
    d.prm.epsilon = (float)resolution;
    d.prm.max_weight = 10000.0f;
    d.prm.is3d = is3d;
    d.win.is3d = is3d;
    for (int k = 0; k < 3; ++k) {
        d.win.dim[k] = dim[k];
        const double c = center ? center[k] : 0.0;
        d.win.base[k] = (k < 2 || is3d) ? (int32_t)(w2m(c, d.prm.scale) >> kPatchLog2) - dim[k] / 2 : 0;
    }
    d.log2v = is3d ? 3 * kPatchLog2 : 2 * kPatchLog2;
    d.ndir = (int)ndir;
    d.pool = pool;
    d.h_dir.assign((size_t)ndir, -1);
    auto bail = [&](const std::string& m) -> TsdmDev* { err = m; delete t; return nullptr; };
#define TS_NEW(expr)                                                                          \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) return bail(std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)
    TS_NEW(cudaSetDevice(dev.device));
    if (dev.stream) {
        d.stream = reinterpret_cast<cudaStream_t>(dev.stream);
    } else {
        TS_NEW(cudaStreamCreateWithFlags(&d.stream, cudaStreamNonBlocking));
        d.own_stream = true;
    }
    TS_NEW(cudaEventCreate(&d.ev[0]));
    TS_NEW(cudaEventCreate(&d.ev[1]));
    const size_t per = (size_t)1 << d.log2v;
    TS_NEW(cudaMalloc((void**)&d.dir, (size_t)ndir * 4));
    TS_NEW(cudaMalloc((void**)&d.marks, (size_t)ndir * 4));
    TS_NEW(cudaMalloc((void**)&d.cells, (size_t)pool * per * sizeof(float2)));
    TS_NEW(cudaMalloc((void**)&d.on, (size_t)pool * per / 8));
    TS_NEW(cudaMalloc((void**)&d.status, 4));
    TS_NEW(cudaMemcpyAsync(d.dir, d.h_dir.data(), (size_t)ndir * 4, cudaMemcpyHostToDevice, d.stream));
    const McTable mc = mc_build_table();
    TS_NEW(cudaMemcpyToSymbolAsync(c_mc_tri, mc.tri, sizeof(mc.tri), 0, cudaMemcpyHostToDevice, d.stream));
    TS_NEW(cudaMemcpyToSymbolAsync(c_mc_ntri, mc.ntri, sizeof(mc.ntri), 0, cudaMemcpyHostToDevice, d.stream));
    TS_NEW(cudaStreamSynchronize(d.stream));
#undef TS_NEW
    return t;
}

TsdmDev::~TsdmDev() { delete d_; }

void TsdmDev::set_max_distance(double dist) { d_->prm.truncate = (float)dist; }
double TsdmDev::max_distance() const { return d_->prm.truncate; }
double TsdmDev::resolution() const { return d_->resolution; }

void TsdmDev::kernel_times(double ms[3], uint64_t launches[3]) const
{
    for (int k = 0; k < 3; ++k) {
        if (ms) ms[k] = d_->ms[k];
        if (launches) launches[k] = d_->launches[k];
    }
}

int TsdmDev::insert_point_clouds(const double* pts, const int64_t* offsets, int n_clouds, const double* origins, const double* quats, uint64_t* inserted)
{
    Impl& d = *d_;
    if (n_clouds < 0) { err_ = "negative number of clouds"; return LAMA_ERR_ARG; }
    if (n_clouds == 0) return LAMA_OK;
    if (!offsets || offsets[0] != 0) { err_ = "offsets must start at 0"; return LAMA_ERR_ARG; }
    for (int k = 0; k < n_clouds; ++k)
        if (offsets[k + 1] < offsets[k]) { err_ = "offsets must not decrease"; return LAMA_ERR_ARG; }
    const int64_t n_pts = offsets[n_clouds];
    if (n_pts > 0 && !pts) { err_ = "null points"; return LAMA_ERR_ARG; }
    if (n_pts >= (int64_t)1 << 40) { err_ = "too many points"; return LAMA_ERR_ARG; }
    TS_TRY(cudaSetDevice(d.device));
    if (d.timing) TS_TRY(cudaEventRecord(d.ev[0], d.stream));
    std::vector<Affine> tf((size_t)n_clouds);
    for (int k = 0; k < n_clouds; ++k) {
        const MovingTf m = moving_tf(origins ? origins + 3 * k : nullptr, quats ? quats + 4 * k : nullptr);
        std::memcpy(tf[k].l, m.l, sizeof(m.l));
        std::memcpy(tf[k].t, m.t, sizeof(m.t));
    }
    TS_TRY(d.ensure(d.pts, std::max<size_t>(1, (size_t)n_pts * 24)));
    TS_TRY(d.ensure(d.off, (size_t)(n_clouds + 1) * 8));
    TS_TRY(d.ensure(d.tf, (size_t)n_clouds * sizeof(Affine)));
    TS_TRY(d.ensure(d.surv, std::max<size_t>(1, (size_t)n_pts)));
    TS_TRY(d.ensure(d.counts, (size_t)(n_pts + 1) * 8));
    TS_TRY(d.ensure(d.offs, (size_t)(n_pts + 1) * 8));
    TS_TRY(d.ensure(d.inserted, (size_t)n_clouds * 4));
    TS_TRY(d.ensure(d.bound, (size_t)(n_clouds + 1) * 8));
    if (n_pts) TS_TRY(cudaMemcpyAsync(d.pts.p, pts, (size_t)n_pts * 24, cudaMemcpyHostToDevice, d.stream));
    TS_TRY(cudaMemcpyAsync(d.off.p, offsets, (size_t)(n_clouds + 1) * 8, cudaMemcpyHostToDevice, d.stream));
    TS_TRY(cudaMemcpyAsync(d.tf.p, tf.data(), (size_t)n_clouds * sizeof(Affine), cudaMemcpyHostToDevice, d.stream));
    TS_TRY(cudaMemsetAsync(d.inserted.p, 0, (size_t)n_clouds * 4, d.stream));
    TS_TRY(cudaMemsetAsync(d.status, 0, 4, d.stream));
    TS_TRY(cudaMemsetAsync(d.marks, 0, (size_t)d.ndir * 4, d.stream));
    TS_TRY(cudaMemsetAsync((uint64_t*)d.counts.p + n_pts, 0, 8, d.stream));

    const View v = d.view();
    FuseParams f{};
    f.pts = (const double*)d.pts.p;
    f.offsets = (const int64_t*)d.off.p;
    f.tf = (const Affine*)d.tf.p;
    f.n_clouds = n_clouds;
    f.prm = d.prm;
    f.surv = (uint8_t*)d.surv.p;
    f.counts = (uint64_t*)d.counts.p;
    f.offs = (const uint64_t*)d.offs.p;
    f.marks = d.marks;
    f.inserted = (uint32_t*)d.inserted.p;
    f.status = d.status;

    // 1-2. dedupe, window check, marks and counts, in passes of whole clouds
    for (int c0 = 0; c0 < n_clouds;) {
        int c1 = c0 + 1;
        while (c1 < n_clouds && c1 - c0 < kHashClouds && offsets[c1 + 1] - offsets[c0] <= kHashPoints) ++c1;
        const int64_t np = offsets[c1] - offsets[c0];
        if (np > 0) {
            uint32_t cap = 1024;
            while ((int64_t)cap < 2 * np) cap <<= 1;
            TS_TRY(d.ensure(d.hkeys, (size_t)cap * 8));
            TS_TRY(d.ensure(d.hval, (size_t)cap * 4));
            TS_TRY(d.ensure(d.hslot, (size_t)np * 4));
            TS_TRY(cudaMemsetAsync(d.hkeys.p, 0xFF, (size_t)cap * 8, d.stream));
            TS_TRY(cudaMemsetAsync(d.hval.p, 0xFF, (size_t)cap * 4, d.stream));
            f.hkeys = (uint64_t*)d.hkeys.p;
            f.hval = (uint32_t*)d.hval.p;
            f.hmask = cap - 1;
            f.hslot = (uint32_t*)d.hslot.p;
            f.p0 = offsets[c0];
            f.p1 = offsets[c1];
            f.c0 = c0;
            k_tsdm_hash<<<blocks_for(np), kThreads, 0, d.stream>>>(f, v);
            k_tsdm_walk<false><<<blocks_for(np), kThreads, 0, d.stream>>>(f, v);
            d.launches[0] += 2;
        }
        c0 = c1;
    }
    TS_TRY(cudaGetLastError());
    uint32_t status = 0;
    TS_TRY(cudaMemcpyAsync(&status, d.status, 4, cudaMemcpyDeviceToHost, d.stream));
    std::vector<uint32_t> marks((size_t)d.ndir);
    TS_TRY(cudaMemcpyAsync(marks.data(), d.marks, (size_t)d.ndir * 4, cudaMemcpyDeviceToHost, d.stream));
    TS_TRY(cudaStreamSynchronize(d.stream));
    if (status & kErrWindow) { err_ = "a hit or ray cell lies outside the directory window"; return LAMA_ERR_WINDOW; }

    // 3. allocate the marked patches, ascending directory index
    std::vector<int32_t> fresh;
    for (int i = 0; i < d.ndir; ++i)
        if (marks[i] && d.h_dir[i] < 0) fresh.push_back(i);
    if ((int64_t)d.used + (int64_t)fresh.size() > d.pool) { err_ = "the patch pool is exhausted (raise pool_slots)"; return LAMA_ERR_POOL; }
    if (!fresh.empty()) {
        std::vector<int32_t> slots(fresh.size());
        for (size_t i = 0; i < fresh.size(); ++i) d.h_dir[fresh[i]] = slots[i] = d.used++;
        TS_TRY(d.ensure(d.slots, slots.size() * 4));
        TS_TRY(cudaMemcpyAsync(d.slots.p, slots.data(), slots.size() * 4, cudaMemcpyHostToDevice, d.stream));
        TS_TRY(cudaMemcpyAsync(d.dir, d.h_dir.data(), (size_t)d.ndir * 4, cudaMemcpyHostToDevice, d.stream));
        k_tsdm_zero<<<std::min<uint64_t>(4096, blocks_for(slots.size() << d.log2v)), kThreads, 0, d.stream>>>((const int32_t*)d.slots.p, (int)slots.size(), v);
        d.launches[0] += 1;
    }

    // 4. record offsets, chunk bounds at cloud boundaries
    size_t scan_bytes = 0;
    TS_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint64_t*)d.counts.p, (uint64_t*)d.offs.p, (int64_t)(n_pts + 1), d.stream));
    TS_TRY(d.ensure(d.temp, scan_bytes));
    TS_TRY(cub::DeviceScan::ExclusiveSum(d.temp.p, scan_bytes, (const uint64_t*)d.counts.p, (uint64_t*)d.offs.p, (int64_t)(n_pts + 1), d.stream));
    k_tsdm_gather<<<blocks_for(n_clouds + 1), kThreads, 0, d.stream>>>((const uint64_t*)d.offs.p, f.offsets, n_clouds + 1, (uint64_t*)d.bound.p);
    std::vector<uint64_t> bound((size_t)n_clouds + 1);
    TS_TRY(cudaMemcpyAsync(bound.data(), d.bound.p, bound.size() * 8, cudaMemcpyDeviceToHost, d.stream));
    TS_TRY(cudaStreamSynchronize(d.stream));

    int end_bit = d.log2v;
    while ((1ll << (end_bit - d.log2v)) < d.ndir) ++end_bit;
    for (int c0 = 0; c0 < n_clouds;) {
        int c1 = c0 + 1;
        while (c1 < n_clouds && bound[c1 + 1] - bound[c0] <= kRecordCap) ++c1;
        const uint64_t nrec = bound[c1] - bound[c0];
        const int64_t np = offsets[c1] - offsets[c0];
        if (np > 0) {
            for (int b = 0; b < 2; ++b) {
                TS_TRY(d.ensure(d.rk[b], std::max<uint64_t>(1, nrec) * 8));
                TS_TRY(d.ensure(d.rv[b], std::max<uint64_t>(1, nrec) * 8));
            }
            f.p0 = offsets[c0];
            f.p1 = offsets[c1];
            f.rec_base = bound[c0];
            f.rkeys = (uint64_t*)d.rk[0].p;
            f.rvals = (uint64_t*)d.rv[0].p;
            k_tsdm_walk<true><<<blocks_for(np), kThreads, 0, d.stream>>>(f, v);
            d.launches[0] += 1;
        }
        if (nrec > 0) {
            size_t sort_bytes = 0;
            TS_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t*)d.rk[0].p, (uint64_t*)d.rk[1].p, (const uint64_t*)d.rv[0].p,
                                                   (uint64_t*)d.rv[1].p, (int64_t)nrec, 0, end_bit, d.stream));
            TS_TRY(d.ensure(d.temp, sort_bytes));
            TS_TRY(cub::DeviceRadixSort::SortPairs(d.temp.p, sort_bytes, (const uint64_t*)d.rk[0].p, (uint64_t*)d.rk[1].p, (const uint64_t*)d.rv[0].p,
                                                   (uint64_t*)d.rv[1].p, (int64_t)nrec, 0, end_bit, d.stream));
            k_tsdm_fold<<<blocks_for(nrec), kThreads, 0, d.stream>>>((const uint64_t*)d.rk[1].p, (const uint64_t*)d.rv[1].p, nrec, v, d.prm.max_weight);
            d.launches[0] += 2;
        }
        c0 = c1;
    }
    TS_TRY(cudaGetLastError());
    std::vector<uint32_t> ins((size_t)n_clouds);
    TS_TRY(cudaMemcpyAsync(ins.data(), d.inserted.p, ins.size() * 4, cudaMemcpyDeviceToHost, d.stream));
    if (d.timing) TS_TRY(cudaEventRecord(d.ev[1], d.stream));
    TS_TRY(cudaStreamSynchronize(d.stream));
    if (d.timing) {
        float t = 0;
        TS_TRY(cudaEventElapsedTime(&t, d.ev[0], d.ev[1]));
        d.ms[0] += t;
    }
    if (inserted)
        for (int k = 0; k < n_clouds; ++k) inserted[k] = ins[k];
    return LAMA_OK;
}

int TsdmDev::distance(const double* pts, int n, double* dist, double* grad)
{
    Impl& d = *d_;
    if (n < 0 || (n > 0 && (!pts || !dist))) { err_ = "null argument"; return LAMA_ERR_ARG; }
    if (n == 0) return LAMA_OK;
    TS_TRY(cudaSetDevice(d.device));
    TS_TRY(d.ensure(d.pts, (size_t)n * 24));
    TS_TRY(d.ensure(d.qout, (size_t)n * 32));
    TS_TRY(cudaMemcpyAsync(d.pts.p, pts, (size_t)n * 24, cudaMemcpyHostToDevice, d.stream));
    double* dd = (double*)d.qout.p;
    if (d.timing) TS_TRY(cudaEventRecord(d.ev[0], d.stream));
    k_tsdm_distance<<<blocks_for(n), kThreads, 0, d.stream>>>((const double*)d.pts.p, n, d.view(), d.prm, dd, dd + n);
    d.launches[1] += 1;
    if (d.timing) TS_TRY(cudaEventRecord(d.ev[1], d.stream));
    TS_TRY(cudaGetLastError());
    TS_TRY(cudaMemcpyAsync(dist, dd, (size_t)n * 8, cudaMemcpyDeviceToHost, d.stream));
    if (grad) TS_TRY(cudaMemcpyAsync(grad, dd + n, (size_t)n * 24, cudaMemcpyDeviceToHost, d.stream));
    TS_TRY(cudaStreamSynchronize(d.stream));
    if (d.timing) {
        float t = 0;
        TS_TRY(cudaEventElapsedTime(&t, d.ev[0], d.ev[1]));
        d.ms[1] += t;
    }
    return LAMA_OK;
}

// Map::bounds (map.cpp:139-157) in 3-D: the anchors of the allocated patches, max + patch_length on every axis
int TsdmDev::bounds(uint32_t mn[3], uint32_t mx[3], int* patches) const
{
    const Impl& d = *d_;
    int n = 0;
    for (int k = 0; k < 3; ++k) { mn[k] = 0xFFFFFFFFu; mx[k] = 0; }
    for (int i = 0; i < d.ndir; ++i) {
        if (d.h_dir[i] < 0) continue;
        const int p[3] = {i % d.win.dim[0], (i / d.win.dim[0]) % d.win.dim[1], i / (d.win.dim[0] * d.win.dim[1])};
        for (int k = 0; k < 3; ++k) {
            const uint32_t a = (k < 2 || d.win.is3d) ? (uint32_t)(d.win.base[k] + p[k]) << kPatchLog2 : 0u;
            mn[k] = std::min(mn[k], a);
            mx[k] = std::max(mx[k], a);
        }
        ++n;
    }
    for (int k = 0; k < 3; ++k) mx[k] += kPatchLen;
    if (patches) *patches = n;
    return LAMA_OK;
}

int TsdmDev::export_box(const uint32_t lo[3], const int32_t size[3], float* dist, float* weight, uint8_t* on)
{
    Impl& d = *d_;
    if (size[0] < 1 || size[1] < 1 || size[2] < 1) { err_ = "empty box"; return LAMA_ERR_ARG; }
    const size_t n = (size_t)size[0] * size[1] * size[2];
    TS_TRY(cudaSetDevice(d.device));
    TS_TRY(d.ensure(d.box[0], n * 4));
    TS_TRY(d.ensure(d.box[1], n * 4));
    TS_TRY(d.ensure(d.box[2], n));
    k_tsdm_export<<<std::min<uint64_t>(8192, blocks_for(n)), kThreads, 0, d.stream>>>(d.view(), lo[0], lo[1], lo[2], size[0], size[1], size[2],
                                                                                      (float*)d.box[0].p, (float*)d.box[1].p, (uint8_t*)d.box[2].p);
    TS_TRY(cudaGetLastError());
    if (dist) TS_TRY(cudaMemcpyAsync(dist, d.box[0].p, n * 4, cudaMemcpyDeviceToHost, d.stream));
    if (weight) TS_TRY(cudaMemcpyAsync(weight, d.box[1].p, n * 4, cudaMemcpyDeviceToHost, d.stream));
    if (on) TS_TRY(cudaMemcpyAsync(on, d.box[2].p, n, cudaMemcpyDeviceToHost, d.stream));
    TS_TRY(cudaStreamSynchronize(d.stream));
    return LAMA_OK;
}

int TsdmDev::to_mesh(float* vertices, size_t cap, size_t* n_vertices)
{
    Impl& d = *d_;
    std::vector<int32_t> list;
    for (int i = 0; i < d.ndir; ++i)
        if (d.h_dir[i] >= 0) list.push_back(i);
    if (list.empty()) {
        if (n_vertices) *n_vertices = 0;
        return LAMA_OK;
    }
    TS_TRY(cudaSetDevice(d.device));
    const uint64_t total = (uint64_t)list.size() << d.log2v;
    TS_TRY(d.ensure(d.list, list.size() * 4));
    TS_TRY(d.ensure(d.counts, (total + 1) * 8));
    TS_TRY(d.ensure(d.offs, (total + 1) * 8));
    TS_TRY(cudaMemcpyAsync(d.list.p, list.data(), list.size() * 4, cudaMemcpyHostToDevice, d.stream));
    TS_TRY(cudaMemsetAsync((uint64_t*)d.counts.p + total, 0, 8, d.stream));
    if (d.timing) TS_TRY(cudaEventRecord(d.ev[0], d.stream));
    const View v = d.view();
    k_tsdm_mesh<false><<<blocks_for(total), kThreads, 0, d.stream>>>((const int32_t*)d.list.p, (int)list.size(), v, d.prm.scale, (uint64_t*)d.counts.p,
                                                                     nullptr, nullptr);
    size_t scan_bytes = 0;
    TS_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint64_t*)d.counts.p, (uint64_t*)d.offs.p, (int64_t)(total + 1), d.stream));
    TS_TRY(d.ensure(d.temp, scan_bytes));
    TS_TRY(cub::DeviceScan::ExclusiveSum(d.temp.p, scan_bytes, (const uint64_t*)d.counts.p, (uint64_t*)d.offs.p, (int64_t)(total + 1), d.stream));
    uint64_t nv = 0;
    TS_TRY(cudaMemcpyAsync(&nv, (uint64_t*)d.offs.p + total, 8, cudaMemcpyDeviceToHost, d.stream));
    TS_TRY(cudaStreamSynchronize(d.stream));
    d.launches[2] += 2;
    if (n_vertices) *n_vertices = (size_t)nv;
    if (!vertices || cap < nv || nv == 0) return LAMA_OK;
    TS_TRY(d.ensure(d.mesh, (size_t)nv * 12));
    k_tsdm_mesh<true><<<blocks_for(total), kThreads, 0, d.stream>>>((const int32_t*)d.list.p, (int)list.size(), v, d.prm.scale, nullptr,
                                                                    (const uint64_t*)d.offs.p, (float*)d.mesh.p);
    d.launches[2] += 1;
    if (d.timing) TS_TRY(cudaEventRecord(d.ev[1], d.stream));
    TS_TRY(cudaGetLastError());
    TS_TRY(cudaMemcpyAsync(vertices, d.mesh.p, (size_t)nv * 12, cudaMemcpyDeviceToHost, d.stream));
    TS_TRY(cudaStreamSynchronize(d.stream));
    if (d.timing) {
        float t = 0;
        TS_TRY(cudaEventElapsedTime(&t, d.ev[0], d.ev[1]));
        d.ms[2] += t;
    }
    return LAMA_OK;
}

}  // namespace lama_b200
