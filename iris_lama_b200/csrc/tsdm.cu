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
//   3. The host allocates the marked patches (ascending directory index) from the pool; k_patch_zero clears them.
//   4. An exclusive scan of the counts gives every point its first record, in (cloud, point, step) order.  The batch is cut at
//      cloud boundaries into chunks of at most kRecordCap records; per chunk k_tsdm_walk<true> sets the "on" bits of every walked
//      voxel (skipped ones too, as the reference's mutable get() does) and writes the records, a stable radix sort orders them by
//      cell, and k_fold_runs folds each run of equal keys in record order, loading and storing its cell once.
// Steps 3 and 4 and the store itself are patch_store.cuh, shared with the 3-D occupancy maps.
#include "mc_table.h"
#include "patch_store.cuh"
#include "tsdm.h"
#include "tsdm_core.h"

namespace lama_b200 {

namespace {

constexpr int64_t kHashPoints = 1 << 20;               // points of one dedupe pass (the hash has >= 2x as many slots)
constexpr int kHashClouds = 65535;                      // clouds of one dedupe pass (16 bits of the hash key)

__constant__ int8_t c_mc_tri[256][kMcRow];
__constant__ uint8_t c_mc_ntri[256];

struct View {
    const int32_t* dir;   // slot of each directory entry, -1 = absent
    float2* cells;        // pool: {distance, weight} per cell
    uint32_t* mask;       // pool: the "on" bit of each cell
    PatchWindow w;
    int log2v;            // log2 of the cells of a patch: 10 (2-D) or 15 (3-D)
};

// the const get() (map.cpp:414-455): false when the patch is absent or the cell is off
__device__ __forceinline__ bool cell_get(const View& v, uint32_t x, uint32_t y, uint32_t z, float2& out)
{
    const int64_t g = cell_pool_index(v.w, v.dir, v.log2v, x, y, z);
    if (g < 0 || !((v.mask[g >> 5] >> (g & 31)) & 1u)) return false;
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
    const PatchWindow& w = v.w;
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
        const int di = window_dir_index(v.w, w.x, w.y, w.z);
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
            const uint32_t ci = window_cell_index(w.x, w.y, w.z, v.w.is3d);
            const size_t g = pool_index(v, v.dir[di], ci);
            atomicOr(&v.mask[g >> 5], 1u << (g & 31));
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

// k_fold_runs' fold of one record into its cell
struct RecordFold {
    static __device__ __forceinline__ void fold(float2& cell, uint64_t r, float max_weight)
    {
        tsdm_fold(cell.x, cell.y, __uint_as_float((uint32_t)r), __uint_as_float((uint32_t)(r >> 32)), max_weight);
    }
};

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

// k_export_box's cell: distance, weight and the "on" bit, zeros where the const get() returns nothing
struct BoxCell {
    static constexpr int kPlanes = 3;
    static constexpr size_t kBytes[kPlanes] = {4, 4, 1};
    static __device__ __forceinline__ void put(const View& v, int64_t g, size_t i, const Planes& out)
    {
        const bool on = g >= 0 && ((v.mask[g >> 5] >> (g & 31)) & 1u);
        const float2 c = on ? v.cells[g] : make_float2(0.f, 0.f);
        ((float*)out.p[0])[i] = c.x;
        ((float*)out.p[1])[i] = c.y;
        ((uint8_t*)out.p[2])[i] = on;
    }
};

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
    if ((v.mask[g >> 5] >> (g & 31)) & 1u) {   // visit_all_cells: every "on" cell, at p2m(patch) + c2m(cell)
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

}  // namespace

// ---- host side ----------------------------------------------------------------------------------------------------------------
struct TsdmDev::Impl : PatchStore {
    double resolution = 0;
    TsdmParams prm{};
    Buf hkeys, hval, hslot, surv, inserted, qout, list, mesh;

    ~Impl() { quiesce(); }

    View view() const { return View{dir, (float2*)cells, mask, win, log2v}; }
};

TsdmDev* TsdmDev::create(double resolution, uint32_t patch_size, bool is3d, const double center[3], const int32_t window[3], const DeviceOptions& dev,
                         std::string& err, int* code)
{
    const int32_t dim2d[3] = {dev.dir_dim, dev.dir_dim, 1};
    PatchWindow win;
    *code = PatchStore::make_window(resolution, patch_size, window, is3d ? kWindow3D : dim2d, center, is3d, 1 << 22, win, err);
    if (*code != LAMA_OK) return nullptr;

    TsdmDev* t = new TsdmDev();
    t->d_ = new Impl();
    Impl& d = *t->d_;
    d.resolution = resolution;
    d.prm.scale = 1.0 / resolution;
    d.prm.truncate = 0.15f;
    d.prm.delta = (float)(4 * resolution);
    d.prm.epsilon = (float)resolution;
    d.prm.max_weight = 10000.0f;
    d.prm.is3d = is3d;
    *code = d.init(dev, win, is3d ? 3 * kPatchLog2 : 2 * kPatchLog2, sizeof(float2), err);
    if (*code != LAMA_OK) { delete t; return nullptr; }
    const McTable mc = mc_build_table();
    cudaError_t e = cudaMemcpyToSymbolAsync(c_mc_tri, mc.tri, sizeof(mc.tri), 0, cudaMemcpyHostToDevice, d.stream);
    if (e == cudaSuccess) e = cudaMemcpyToSymbolAsync(c_mc_ntri, mc.ntri, sizeof(mc.ntri), 0, cudaMemcpyHostToDevice, d.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(d.stream);
    if (e != cudaSuccess) {
        err = std::string("marching-cubes table: ") + cudaGetErrorString(e);
        *code = PatchStore::cuda_failure();
        delete t;
        return nullptr;
    }
    return t;
}

TsdmDev::~TsdmDev() { delete d_; }

void TsdmDev::set_max_distance(double dist) { d_->prm.truncate = (float)dist; }
double TsdmDev::max_distance() const { return d_->prm.truncate; }
double TsdmDev::resolution() const { return d_->resolution; }
void TsdmDev::kernel_times(double ms[3], uint64_t launches[3]) const { d_->kernel_times(ms, launches); }

int TsdmDev::insert_point_clouds(const double* pts, const int64_t* offsets, int n_clouds, const double* origins, const double* quats, uint64_t* inserted)
{
    Impl& d = *d_;
    int64_t n_pts = 0;
    int rc = PatchStore::check_clouds(pts, offsets, n_clouds, n_pts, err_);
    if (rc != LAMA_OK || n_clouds == 0) return rc;
    PS_TRY(cudaSetDevice(d.device));
    PS_TRY(d.record(0));
    PS_TRY(d.upload_clouds(pts, offsets, n_clouds, n_pts, origins, quats));
    PS_TRY(d.surv.reserve(std::max<size_t>(1, (size_t)n_pts)));
    PS_TRY(d.inserted.reserve((size_t)n_clouds * 4));
    PS_TRY(cudaMemsetAsync(d.inserted.get(), 0, (size_t)n_clouds * 4, d.stream));

    const View v = d.view();
    FuseParams f{};
    f.pts = (const double*)d.pts.get();
    f.offsets = (const int64_t*)d.off.get();
    f.tf = (const Affine*)d.tf.get();
    f.n_clouds = n_clouds;
    f.prm = d.prm;
    f.surv = (uint8_t*)d.surv.get();
    f.counts = (uint64_t*)d.counts.get();
    f.offs = (const uint64_t*)d.offs.get();
    f.marks = d.marks;
    f.inserted = (uint32_t*)d.inserted.get();
    f.status = d.status;

    // 1-2. dedupe, window check, marks and counts, in passes of whole clouds
    for (int c0 = 0; c0 < n_clouds;) {
        int c1 = c0 + 1;
        while (c1 < n_clouds && c1 - c0 < kHashClouds && offsets[c1 + 1] - offsets[c0] <= kHashPoints) ++c1;
        const int64_t np = offsets[c1] - offsets[c0];
        if (np > 0) {
            uint32_t cap = 1024;
            while ((int64_t)cap < 2 * np) cap <<= 1;
            PS_TRY(d.hkeys.reserve((size_t)cap * 8));
            PS_TRY(d.hval.reserve((size_t)cap * 4));
            PS_TRY(d.hslot.reserve((size_t)np * 4));
            PS_TRY(cudaMemsetAsync(d.hkeys.get(), 0xFF, (size_t)cap * 8, d.stream));
            PS_TRY(cudaMemsetAsync(d.hval.get(), 0xFF, (size_t)cap * 4, d.stream));
            f.hkeys = (uint64_t*)d.hkeys.get();
            f.hval = (uint32_t*)d.hval.get();
            f.hmask = cap - 1;
            f.hslot = (uint32_t*)d.hslot.get();
            f.p0 = offsets[c0];
            f.p1 = offsets[c1];
            f.c0 = c0;
            k_tsdm_hash<<<blocks_for(np), kThreads, 0, d.stream>>>(f, v);
            k_tsdm_walk<false><<<blocks_for(np), kThreads, 0, d.stream>>>(f, v);
            d.launches[0] += 2;
        }
        c0 = c1;
    }
    PS_TRY(cudaGetLastError());
    uint32_t status = 0;
    std::vector<uint32_t> marks;
    PS_TRY(d.read_marks(status, marks));
    if (status & kErrWindow) { err_ = "a hit or ray cell lies outside the directory window"; return LAMA_ERR_WINDOW; }

    // 3. allocate the marked patches, ascending directory index
    rc = d.alloc_marked(marks, v, err_, d.launches[0]);
    if (rc != LAMA_OK) return rc;

    // 4. record offsets, chunk bounds at cloud boundaries
    std::vector<uint64_t> bound;
    PS_TRY(d.scan_records(n_pts, n_clouds, bound));
    rc = PatchStore::for_each_chunk(bound, n_clouds, [&](int c0, int c1, uint64_t nrec) -> int {
        const int64_t np = offsets[c1] - offsets[c0];
        if (np > 0) {   // also without records: the walk turns the skipped voxels on
            PS_TRY(d.ensure_records<uint64_t>(nrec));
            f.p0 = offsets[c0];
            f.p1 = offsets[c1];
            f.rec_base = bound[c0];
            f.rkeys = (uint64_t*)d.rk[0].get();
            f.rvals = (uint64_t*)d.rv[0].get();
            k_tsdm_walk<true><<<blocks_for(np), kThreads, 0, d.stream>>>(f, v);
            d.launches[0] += 1;
        }
        if (nrec > 0) {
            PS_TRY(d.sort_fold<uint64_t, RecordFold>((int64_t)nrec, v, d.prm.max_weight));
            d.launches[0] += 2;
        }
        return LAMA_OK;
    });
    if (rc != LAMA_OK) return rc;
    PS_TRY(cudaGetLastError());
    std::vector<uint32_t> ins((size_t)n_clouds);
    PS_TRY(cudaMemcpyAsync(ins.data(), d.inserted.get(), ins.size() * 4, cudaMemcpyDeviceToHost, d.stream));
    PS_TRY(d.record(1));
    PS_TRY(d.finish(0));
    if (inserted)
        for (int k = 0; k < n_clouds; ++k) inserted[k] = ins[k];
    return LAMA_OK;
}

int TsdmDev::distance(const double* pts, int n, double* dist, double* grad)
{
    Impl& d = *d_;
    if (n < 0 || (n > 0 && (!pts || !dist))) { err_ = "null argument"; return LAMA_ERR_ARG; }
    if (n == 0) return LAMA_OK;
    PS_TRY(cudaSetDevice(d.device));
    PS_TRY(d.pts.reserve((size_t)n * 24));
    PS_TRY(d.qout.reserve((size_t)n * 32));
    PS_TRY(cudaMemcpyAsync(d.pts.get(), pts, (size_t)n * 24, cudaMemcpyHostToDevice, d.stream));
    double* dd = (double*)d.qout.get();
    PS_TRY(d.record(0));
    k_tsdm_distance<<<blocks_for(n), kThreads, 0, d.stream>>>((const double*)d.pts.get(), n, d.view(), d.prm, dd, dd + n);
    d.launches[1] += 1;
    PS_TRY(d.record(1));
    PS_TRY(cudaGetLastError());
    PS_TRY(cudaMemcpyAsync(dist, dd, (size_t)n * 8, cudaMemcpyDeviceToHost, d.stream));
    if (grad) PS_TRY(cudaMemcpyAsync(grad, dd + n, (size_t)n * 24, cudaMemcpyDeviceToHost, d.stream));
    PS_TRY(d.finish(1));
    return LAMA_OK;
}

int TsdmDev::bounds(uint32_t mn[3], uint32_t mx[3], int* patches) const
{
    d_->bounds(mn, mx, patches);
    return LAMA_OK;
}

int TsdmDev::export_box(const uint32_t lo[3], const int32_t size[3], float* dist, float* weight, uint8_t* on)
{
    void* const host[] = {dist, weight, on};
    return d_->export_box<BoxCell>(d_->view(), lo, size, host, err_);
}

int TsdmDev::to_mesh(float* vertices, size_t cap, size_t* n_vertices)
{
    Impl& d = *d_;
    const std::vector<int32_t> list = d.allocated();
    if (list.empty()) {
        if (n_vertices) *n_vertices = 0;
        return LAMA_OK;
    }
    PS_TRY(cudaSetDevice(d.device));
    const uint64_t total = (uint64_t)list.size() << d.log2v;
    PS_TRY(d.list.reserve(list.size() * 4));
    PS_TRY(d.counts.reserve((total + 1) * 8));
    PS_TRY(d.offs.reserve((total + 1) * 8));
    PS_TRY(cudaMemcpyAsync(d.list.get(), list.data(), list.size() * 4, cudaMemcpyHostToDevice, d.stream));
    PS_TRY(cudaMemsetAsync((uint64_t*)d.counts.get() + total, 0, 8, d.stream));
    PS_TRY(d.record(0));
    const View v = d.view();
    k_tsdm_mesh<false><<<blocks_for(total), kThreads, 0, d.stream>>>((const int32_t*)d.list.get(), (int)list.size(), v, d.prm.scale, (uint64_t*)d.counts.get(),
                                                                     nullptr, nullptr);
    PS_TRY(d.scan_counts((int64_t)(total + 1)));
    uint64_t nv = 0;
    PS_TRY(cudaMemcpyAsync(&nv, (uint64_t*)d.offs.get() + total, 8, cudaMemcpyDeviceToHost, d.stream));
    PS_TRY(cudaStreamSynchronize(d.stream));
    d.launches[2] += 2;
    if (n_vertices) *n_vertices = (size_t)nv;
    if (!vertices || cap < nv || nv == 0) return LAMA_OK;
    PS_TRY(d.mesh.reserve((size_t)nv * 12));
    k_tsdm_mesh<true><<<blocks_for(total), kThreads, 0, d.stream>>>((const int32_t*)d.list.get(), (int)list.size(), v, d.prm.scale, nullptr,
                                                                    (const uint64_t*)d.offs.get(), (float*)d.mesh.get());
    d.launches[2] += 1;
    PS_TRY(d.record(1));
    PS_TRY(cudaGetLastError());
    PS_TRY(cudaMemcpyAsync(vertices, d.mesh.get(), (size_t)nv * 12, cudaMemcpyDeviceToHost, d.stream));
    PS_TRY(d.finish(2));
    return LAMA_OK;
}

}  // namespace lama_b200
