// om3d.cu -- lama::FrequencyOccupancyMap and lama::ProbabilisticOccupancyMap with is3d = true on the device: point-cloud insertion
// (the loop body of GraphSlam2D::generateOccupancyMap, graph_slam2d.cpp:146-158), ordered per-cell setters, queries, prune, exports
// and 3-D .sdm files.
//
// Insertion, frequency maps.  Every update is a counter increment and increments commute, so the map is built as the 2-D render
// (k_render_scans) builds it:
//   1. k_om3_points<0> (mark): one thread per point, the lanes of a warp on consecutive points.  The thread walks its hit and its ray, checks
//      the window, marks the touched directory entries and counts its updates.  Nothing in the map is written yet: a window error
//      leaves it unchanged.
//   2. The host allocates the marked patches from the pool in ascending directory index (the reference's patch set); k_patch_zero
//      clears them.
//   3. k_om3_points<1> (count) walks again and adds fire-and-forget `red.global.add.u32` reductions.  A hit is a returning add: the hit that
//      finds `occupied` at 0xFFFF takes its carry out of `visited` back.
//   4. k_om3_known sets known |= (word != 0) over the marked entries.
// Insertion, log-odds maps.  Updates are clamped, so their order matters; they are replayed in the reference's order as the TSDM
// fusion does (tsdm.cu): per-point record counts (1 + ray cells) and an exclusive scan place the records in (cloud, point, step)
// order, step 0 being the hit.  The batch is cut at cloud boundaries into chunks of at most kRecordCap records; per chunk
// k_om3_points<2> (emit) writes the records and sets the known bits, a stable radix sort on the cell key groups them by cell (the op travels in
// the value), and k_fold_runs folds each run of equal keys in record order with prob_hit / prob_miss.
// apply() uses the same record -> sort -> fold path for both kinds, with the op's list index in the value.
// The store, the patch allocation, the scan, the chunks and the sort and fold are patch_store.cuh, shared with the TSDM.
#include "om3d.h"
#include "occ_dist3_core.h"
#include "om3d_core.h"
#include "patch_store.cuh"
#include "sdm_io.h"

namespace lama_b200 {

namespace {

struct View {
    static constexpr int log2v = kOm3Log2Cells;
    const int32_t* dir;   // slot of each directory entry, -1 = absent
    uint32_t* cells;      // pool: kOm3Cells words per slot
    uint32_t* mask;       // pool: the known bits, kOm3KnownWords words per slot
    PatchWindow w;
};

__device__ __forceinline__ uint32_t cell_index(uint32_t x, uint32_t y, uint32_t z) { return window_cell_index(x, y, z, 1); }

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
    uint32_t* rvals;          // record: its index within the chunk << 2 | op (the index is read by the coupled fold only)
    uint32_t* marks;          // per directory entry: touched by this batch
    uint32_t* status;
    int margin;               // mark pass: the cells a touched cell must lie inside the window (0: inside it)
};

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
        const int di = window_dir_index(v.w, x, y, z);
        if (kPass == 0) {
            if (di < 0 || (f.margin && !dm3_inside(v.w, x, y, z, f.margin))) { bad = true; return; }
            if (di != last_di) {
                last_di = di;
                if (!f.marks[di]) f.marks[di] = 1;
            }
            return;
        }
        const uint32_t ci = cell_index(x, y, z);
        const int slot = v.dir[di];
        if (kPass == 2) {
            const size_t g = pool_index(v, slot, ci);
            atomicOr(&v.mask[g >> 5], 1u << (g & 31));
            f.rkeys[out] = ((uint32_t)di << kOm3Log2Cells) | ci;
            f.rvals[out] = (uint32_t)(out << 2) | op;   // plain insertion folds the op bits only, whatever the chunk's length
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
    uint32_t* kb = v.mask + (size_t)slot * kOm3KnownWords;
    const int lane = threadIdx.x & 31;
    for (int row = threadIdx.x >> 5; row < kOm3KnownWords; row += kThreads / 32) {
        const uint32_t k = __ballot_sync(0xffffffffu, __ldcg(cells + row * 32 + lane) != 0u);
        if (lane == 0 && k) kb[row] |= k;
    }
}

// apply(): kEmit = false: window check and marks; true: known bits and records (value = list index << 2 | op)
template <bool kEmit>
__global__ void __launch_bounds__(kThreads) k_om3_apply(const uint32_t* __restrict__ xyz, const uint8_t* __restrict__ ops, int n, View v,
                                                        uint32_t* marks, uint32_t* status, uint32_t* rkeys, uint32_t* rvals)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    const int di = window_dir_index(v.w, x, y, z);
    if (!kEmit) {
        if (di < 0) atomicOr(status, kErrWindow);
        else if (!marks[di]) marks[di] = 1;
        return;
    }
    const uint32_t ci = cell_index(x, y, z);
    const size_t g = pool_index(v, v.dir[di], ci);
    atomicOr(&v.mask[g >> 5], 1u << (g & 31));
    rkeys[i] = ((uint32_t)di << kOm3Log2Cells) | ci;
    rvals[i] = ((uint32_t)i << 2) | ops[i];
}

// k_fold_runs' fold of one record (an op in bits 0-1) into its cell.  kApply: changed[value >> 2] = the op's return value.
template <bool kApply>
struct OpFold {
    static __device__ __forceinline__ void fold(uint32_t& word, uint32_t r, int kind, const ProbParams& pp, uint8_t* changed)
    {
        const bool ch = om3_op(kind, word, r & 3u, pp);
        if (kApply) changed[r >> 2] = ch;
    }
};

// ---- the coupled insertion (insert_point_clouds_dm3) ----------------------------------------------------------------------------
// the distance map's directory and pool; its window is the occupancy map's, so a record key addresses the same cell in both
struct DmView {
    const int32_t* dir;
    uint64_t* cells;
};

// one thread per run of equal cell keys, as k_fold_runs: folds the run's records into the occupancy word in record order and runs the
// filter (od3_record) from the distance-map cell's obstacle state; flags[index] = its result
__global__ void __launch_bounds__(kThreads) k_od3_fold(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint64_t n, View v,
                                                       int kind, ProbParams pp, DmView dm, uint8_t* flags)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t k = keys[i];
    if (i > 0 && keys[i - 1] == k) return;
    const uint32_t di = k >> kOm3Log2Cells, ci = k & (kOm3Cells - 1);
    const size_t g = pool_index(v, v.dir[di], ci);
    uint32_t word = v.cells[g];
    const int32_t ds = dm.dir[di];
    bool obstacle = ds >= 0 && dm3_obstacle(dm.cells[((size_t)ds << kDm3Log2Cells) | ci]);
    for (uint64_t j = i; j < n && keys[j] == k; ++j) {
        const uint32_t r = vals[j];
        flags[r >> 2] = (uint8_t)od3_record(kind, pp, word, r, obstacle);
    }
    v.cells[g] = word;
}

// per record (record order) with an event: marks the distance map's directory entry
__global__ void __launch_bounds__(kThreads) k_od3_mark(const uint32_t* __restrict__ keys, const uint8_t* __restrict__ flags, uint64_t n, uint32_t* marks)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !(flags[i] & kOd3Event)) return;
    const uint32_t di = keys[i] >> kOm3Log2Cells;
    if (!marks[di]) marks[di] = 1;
}

// per record: push[i] = 1 when it pushes; an event sets the distance-map cell's known bit (the mutable get() of add / removeObstacle)
// and is counted in *events
__global__ void __launch_bounds__(kThreads) k_od3_known(const uint32_t* __restrict__ keys, const uint8_t* __restrict__ flags, uint64_t n, DmView dm,
                                                        uint32_t* push, unsigned long long* events)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t f = i < n ? flags[i] : 0u;
    const unsigned ev = __ballot_sync(0xffffffffu, (f & kOd3Event) != 0);
    if ((threadIdx.x & 31) == 0 && ev) atomicAdd(events, (unsigned long long)__popc(ev));
    if (i >= n) return;
    push[i] = (f & kOd3Push) ? 1u : 0u;
    if (!(f & kOd3Event)) return;
    const uint32_t k = keys[i];
    unsigned long long* c = (unsigned long long*)dm.cells + (((size_t)dm.dir[k >> kOm3Log2Cells] << kDm3Log2Cells) | (k & (kOm3Cells - 1)));
    if (!(*c & kDm3KnownBit)) atomicOr(c, (unsigned long long)kDm3KnownBit);
}

// the pushing records, in record order, into the brushfire's op list (x, y, z, kind) at their exclusive-scan position
__global__ void __launch_bounds__(kThreads) k_od3_ops(const uint32_t* __restrict__ keys, const uint8_t* __restrict__ flags,
                                                      const uint32_t* __restrict__ pos, uint64_t n, PatchWindow w, uint32_t* ops)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t f = flags[i];
    if (!(f & kOd3Push)) return;
    uint32_t* o = ops + (size_t)kDm3OpWords * pos[i];
    dm3_key_cell(w, keys[i], o[0], o[1], o[2]);
    o[3] = (f & kOd3Remove) ? 1u : 0u;
}

// the op list's segment ends: seg_end[j] = the ops of clouds c0 .. c0 + j (bound: every cloud's first record, rec_base that of c0)
__global__ void k_od3_segments(const uint32_t* __restrict__ pos, const uint64_t* __restrict__ bound, int c0, int n, uint64_t rec_base, uint32_t* seg_end)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) seg_end[j] = pos[bound[c0 + 1 + j] - rec_base];
}

// the cells the const get() returns (map.cpp:414-455, container.h:119-123): word and present (patch allocated, known bit set)
__global__ void __launch_bounds__(kThreads) k_om3_gather(const uint32_t* __restrict__ xyz, int n, View v, uint32_t* words, uint8_t* present)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t g = cell_pool_index(v.w, v.dir, kOm3Log2Cells, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    const bool k = g >= 0 && ((v.mask[g >> 5] >> (g & 31)) & 1u);
    words[i] = k ? v.cells[g] : 0u;
    present[i] = k;
}

// k_export_box's cell: the word and the known bit, 0 where there is no patch
struct BoxCell {
    static constexpr int kPlanes = 2;
    static constexpr size_t kBytes[kPlanes] = {4, 1};
    static __device__ __forceinline__ void put(const View& v, int64_t g, size_t i, const Planes& out)
    {
        ((uint32_t*)out.p[0])[i] = g < 0 ? 0u : v.cells[g];
        ((uint8_t*)out.p[1])[i] = g < 0 ? 0 : (v.mask[g >> 5] >> (g & 31)) & 1u;
    }
};

// FrequencyOccupancyMap::prune (frequency_occupancy_map.cpp:149-158) over the known cells of the first n_slots pool slots
__global__ void k_om3_prune(View v, int n_slots)
{
    const size_t total = (size_t)n_slots << kOm3Log2Cells;
    for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
        if (!((v.mask[g >> 5] >> (g & 31)) & 1u)) continue;
        const uint32_t w = v.cells[g];
        const uint32_t p = om3_prune(w);
        if (p != w) v.cells[g] = p;
    }
}

}  // namespace

// ---- host side ----------------------------------------------------------------------------------------------------------------
struct OccMap3Dev::Impl : PatchStore {
    int kind = kOm3Frequency;
    double resolution = 0, scale = 0;
    ProbParams pp{};
    Buf qin, qout, qflag, ops, changed, dops, dseg;

    ~Impl() { quiesce(); }

    View view() const { return View{dir, (uint32_t*)cells, mask, win}; }
};

OccMap3Dev* OccMap3Dev::create(double resolution, uint32_t patch_size, int kind, const double center[3], const int32_t window[3],
                               const DeviceOptions& dev, std::string& err, int* code)
{
    PatchWindow win;
    *code = PatchStore::make_window(resolution, patch_size, window, kWindow3D, center, true, kOm3MaxEntries, win, err);
    if (*code != LAMA_OK) return nullptr;
    if (kind != kOm3Frequency && kind != kOm3LogOdds) {
        err = "kind must be 0 (frequency) or 1 (log-odds)";
        *code = LAMA_ERR_ARG;
        return nullptr;
    }

    OccMap3Dev* t = new OccMap3Dev();
    t->d_ = new Impl();
    Impl& d = *t->d_;
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
    *code = d.init(dev, win, kOm3Log2Cells, 4, err);
    if (*code != LAMA_OK) { delete t; return nullptr; }
    return t;
}

OccMap3Dev::~OccMap3Dev() { delete d_; }

int OccMap3Dev::kind() const { return d_->kind; }
double OccMap3Dev::resolution() const { return d_->resolution; }
void OccMap3Dev::kernel_times(double ms[3], uint64_t launches[3]) const { d_->kernel_times(ms, launches); }

int OccMap3Dev::insert_point_clouds(const double* pts, const int64_t* offsets, int n_clouds, const double* origins, const double* quats, bool full,
                                    uint64_t* cells)
{
    Impl& d = *d_;
    if (cells) *cells = 0;
    int64_t n_pts = 0;
    int rc = PatchStore::check_clouds(pts, offsets, n_clouds, n_pts, err_);
    if (rc != LAMA_OK || n_pts == 0) return rc;
    PS_TRY(cudaSetDevice(d.device));
    PS_TRY(d.record(0));
    PS_TRY(d.upload_clouds(pts, offsets, n_clouds, n_pts, origins, quats));

    const View v = d.view();
    InsertParams f{};
    f.pts = (const double*)d.pts.get();
    f.offsets = (const int64_t*)d.off.get();
    f.tf = (const Affine*)d.tf.get();
    f.n_clouds = n_clouds;
    f.p0 = 0;
    f.p1 = n_pts;
    f.scale = d.scale;
    f.full = full ? 1 : 0;
    f.counts = (uint64_t*)d.counts.get();
    f.offs = (const uint64_t*)d.offs.get();
    f.marks = d.marks;
    f.status = d.status;

    // 1. window check, marks, record counts; the map is not touched
    k_om3_points<0><<<blocks_for(n_pts), kThreads, 0, d.stream>>>(f, v);
    d.launches[0] += 1;
    PS_TRY(cudaGetLastError());
    uint32_t status = 0;
    std::vector<uint32_t> marks;
    PS_TRY(d.read_marks(status, marks));
    if (status & kErrWindow) { err_ = "a hit or ray cell lies outside the directory window"; return LAMA_ERR_WINDOW; }

    // 2. allocate the marked patches, ascending directory index
    rc = d.alloc_marked(marks, v, err_, d.launches[0]);
    if (rc != LAMA_OK) return rc;

    // 3. record offsets (their total is the number of cell updates)
    std::vector<uint64_t> bound;
    PS_TRY(d.scan_records(n_pts, n_clouds, bound));
    d.launches[0] += 2;

    if (d.kind == kOm3Frequency) {
        // 4f. counter reductions, then the known plane of the touched patches
        k_om3_points<1><<<blocks_for(n_pts), kThreads, 0, d.stream>>>(f, v);
        k_om3_known<<<d.ndir, kThreads, 0, d.stream>>>(v, d.marks);
        d.launches[0] += 2;
    } else {
        // 4p. per chunk of whole clouds: records, stable sort on the cell key, one fold per cell
        rc = PatchStore::for_each_chunk(bound, n_clouds, [&](int c0, int c1, uint64_t nrec) -> int {
            if (nrec == 0) return LAMA_OK;
            PS_TRY(d.ensure_records<uint32_t>(nrec));
            f.p0 = offsets[c0];
            f.p1 = offsets[c1];
            f.rec_base = bound[c0];
            f.rkeys = (uint32_t*)d.rk[0].get();
            f.rvals = (uint32_t*)d.rv[0].get();
            k_om3_points<2><<<blocks_for((uint64_t)(f.p1 - f.p0)), kThreads, 0, d.stream>>>(f, v);
            PS_TRY(d.sort_fold<uint32_t, OpFold<false>>((int64_t)nrec, v, d.kind, d.pp, (uint8_t*)nullptr));
            d.launches[0] += 3;
            return LAMA_OK;
        });
        if (rc != LAMA_OK) return rc;
    }
    PS_TRY(cudaGetLastError());
    PS_TRY(d.record(1));
    PS_TRY(d.finish(0));
    if (cells) *cells = bound[n_clouds];
    return LAMA_OK;
}

// The coupled insertion.  Both maps are admitted before either changes: the mark pass checks every hit and ray cell against a margin
// of R + 1 (R = the distance map's reach), then the distance map's pool check (the marked entries dilated by R), then the occupancy
// map's allocation, which refuses a full pool before it writes.  The distance map's queue is then flushed, and per chunk of whole
// clouds:
//   1. k_om3_points<2> emits the records (value = index << 2 | op) and sets the occupancy known bits; a stable sort groups them by cell.
//   2. k_od3_fold folds each cell's run in record order and writes every record's filter flags.
//   3. k_od3_mark marks the distance map's entries of the events; the distance map allocates them (ascending directory index).
//   4. k_od3_known sets their known bits and counts events, a scan places the pushes, k_od3_ops writes the op list in record order and
//      k_od3_segments its per-cloud ends.
//   5. The distance map applies and updates the list cloud by cloud (k_dm3_brushfire, Brushfire3::run_segments).
// The next chunk's fold reads the obstacle state this chunk's ops left.  Each map works on its own stream; the hand-overs are events.
int OccMap3Dev::insert_point_clouds_dm3(DistMap3Dev& dm, const double* pts, const int64_t* offsets, int n_clouds, const double* origins,
                                        const double* quats, bool full, uint64_t* cells, uint32_t* processed, uint64_t counts[2])
{
    Impl& d = *d_;
    if (cells) *cells = 0;
    if (counts) counts[0] = counts[1] = 0;
    if (processed)
        for (int c = 0; c < n_clouds; ++c) processed[c] = 0;
    int64_t n_pts = 0;
    int rc = PatchStore::check_clouds(pts, offsets, n_clouds, n_pts, err_);
    if (rc != LAMA_OK) return rc;
    const DistMap3Dev::Coupling cp = dm.coupling();
    bool same = cp.device == d.device && cp.resolution == d.resolution;
    for (int k = 0; k < 3; ++k) same = same && cp.win.base[k] == d.win.base[k] && cp.win.dim[k] == d.win.dim[k];
    if (!same) { err_ = "the occupancy and distance maps must share device, resolution and window"; return LAMA_ERR_ARG; }
    if (n_clouds == 0) return LAMA_OK;
    std::vector<uint32_t> proc((size_t)n_clouds, 0);
    uint64_t events = 0, pushes = 0;
    PS_TRY(cudaSetDevice(d.device));

    std::vector<uint64_t> bound((size_t)n_clouds + 1, 0);
    const View v = d.view();
    InsertParams f{};
    if (n_pts > 0) {
        PS_TRY(d.record(0));
        PS_TRY(d.upload_clouds(pts, offsets, n_clouds, n_pts, origins, quats));
        f.pts = (const double*)d.pts.get();
        f.offsets = (const int64_t*)d.off.get();
        f.tf = (const Affine*)d.tf.get();
        f.n_clouds = n_clouds;
        f.p0 = 0;
        f.p1 = n_pts;
        f.scale = d.scale;
        f.full = full ? 1 : 0;
        f.counts = (uint64_t*)d.counts.get();
        f.offs = (const uint64_t*)d.offs.get();
        f.marks = d.marks;
        f.status = d.status;
        f.margin = cp.reach + 1;

        // admission: window margin, record counts, both pools; nothing is written before all three pass
        k_om3_points<0><<<blocks_for(n_pts), kThreads, 0, d.stream>>>(f, v);
        d.launches[0] += 1;
        PS_TRY(cudaGetLastError());
        uint32_t status = 0;
        std::vector<uint32_t> marks;
        PS_TRY(d.read_marks(status, marks));
        if (status & kErrWindow) {
            err_ = "a hit or ray cell lies less than " + std::to_string(cp.reach + 1) + " cells (the distance map's reach + 1) inside the directory window";
            return LAMA_ERR_WINDOW;
        }
        PS_TRY(d.scan_records(n_pts, n_clouds, bound));
        d.launches[0] += 2;
        for (int c = 0; c < n_clouds; ++c)
            if (bound[(size_t)c + 1] - bound[(size_t)c] >= (uint64_t(1) << 30)) { err_ = "a cloud has 2^30 cell updates or more"; return LAMA_ERR_ARG; }
        std::vector<uint8_t> next;
        rc = dm.admit_entries(marks, next);
        if (rc != LAMA_OK) { err_ = dm.error(); return rc; }
        rc = d.alloc_marked(marks, v, err_, d.launches[0]);
        if (rc != LAMA_OK) return rc;
        dm.commit_reachable(next);
        PS_TRY(cudaGetLastError());
        PS_TRY(d.record(1));
        PS_TRY(d.finish(0));
    }
    rc = dm.flush();   // queued ops first: they already sit in the reference's heaps
    if (rc != LAMA_OK) { err_ = dm.error(); return rc; }

    Event ev[2];   // [0] distance map -> occupancy map, [1] the reverse
    for (Event& e : ev) PS_TRY(e.create(cudaEventDisableTiming));
    const DmView dv{cp.dir, cp.cells};
    rc = PatchStore::for_each_chunk(bound, n_clouds, [&](int c0, int c1, uint64_t nrec) -> int {
        std::vector<uint32_t> seg_end((size_t)(c1 - c0), 0);
        if (nrec > 0) {
            PS_TRY(d.record(0));
            PS_TRY(d.ensure_records<uint32_t>(nrec + 1));
            PS_TRY(d.changed.reserve((size_t)nrec));
            f.p0 = offsets[c0];
            f.p1 = offsets[c1];
            f.rec_base = bound[(size_t)c0];
            f.rkeys = (uint32_t*)d.rk[0].get();
            f.rvals = (uint32_t*)d.rv[0].get();
            const uint32_t* keys = (const uint32_t*)d.rk[0].get();   // record order
            uint8_t* flags = (uint8_t*)d.changed.get();
            const unsigned nb = blocks_for(nrec);
            k_om3_points<2><<<blocks_for((uint64_t)(f.p1 - f.p0)), kThreads, 0, d.stream>>>(f, v);
            PS_TRY(d.sort_records<uint32_t>((int64_t)nrec));
            k_od3_fold<<<nb, kThreads, 0, d.stream>>>((const uint32_t*)d.rk[1].get(), (const uint32_t*)d.rv[1].get(), nrec, v, d.kind, d.pp, dv, flags);
            PS_TRY(d.clear_marks());
            k_od3_mark<<<nb, kThreads, 0, d.stream>>>(keys, flags, nrec, d.marks);
            d.launches[0] += 4;
            PS_TRY(cudaGetLastError());
            uint32_t status = 0;
            std::vector<uint32_t> marks;
            PS_TRY(d.read_marks(status, marks));
            rc = dm.alloc_entries(marks, ev[0]);
            if (rc != LAMA_OK) { err_ = dm.error(); return rc; }
            PS_TRY(cudaStreamWaitEvent(d.stream, ev[0], 0));
            // the sorted values are spent: rv[0] takes the push flags, rv[1] their exclusive scan (nrec + 1 entries)
            uint32_t* push = (uint32_t*)d.rv[0].get();
            uint32_t* pos = (uint32_t*)d.rv[1].get();
            PS_TRY(d.dseg.reserve((size_t)(c1 - c0) * 4 + 8));
            unsigned long long* ev_count = (unsigned long long*)d.dseg.get();
            uint32_t* dseg_end = (uint32_t*)((char*)d.dseg.get() + 8);
            PS_TRY(cudaMemsetAsync(ev_count, 0, 8, d.stream));
            PS_TRY(cudaMemsetAsync(push + nrec, 0, 4, d.stream));
            k_od3_known<<<nb, kThreads, 0, d.stream>>>(keys, flags, nrec, dv, push, ev_count);
            size_t bytes = 0;
            PS_TRY(cub::DeviceScan::ExclusiveSum(nullptr, bytes, push, pos, (int64_t)nrec + 1, d.stream));
            PS_TRY(d.temp.reserve(bytes));
            PS_TRY(cub::DeviceScan::ExclusiveSum(d.temp.get(), bytes, push, pos, (int64_t)nrec + 1, d.stream));
            k_od3_segments<<<blocks_for((uint64_t)(c1 - c0)), kThreads, 0, d.stream>>>(pos, (const uint64_t*)d.bound.get(), c0, c1 - c0, bound[(size_t)c0], dseg_end);
            d.launches[0] += 3;
            unsigned long long h_events = 0;
            PS_TRY(cudaMemcpyAsync(&h_events, ev_count, 8, cudaMemcpyDeviceToHost, d.stream));
            PS_TRY(cudaMemcpyAsync(seg_end.data(), dseg_end, seg_end.size() * 4, cudaMemcpyDeviceToHost, d.stream));
            PS_TRY(cudaStreamSynchronize(d.stream));
            const uint32_t n_push = seg_end.back();
            PS_TRY(d.dops.reserve((size_t)std::max<uint32_t>(n_push, 1) * kDm3OpWords * 4));
            k_od3_ops<<<nb, kThreads, 0, d.stream>>>(keys, flags, pos, nrec, d.win, (uint32_t*)d.dops.get());
            d.launches[0] += 1;
            PS_TRY(cudaGetLastError());
            PS_TRY(d.record(1));
            PS_TRY(cudaEventRecord(ev[1], d.stream));
            PS_TRY(d.finish(0));
            events += h_events;
            pushes += n_push;
        }
        rc = dm.run_segments((const uint32_t*)d.dops.get(), seg_end, proc.data() + c0, nrec > 0 ? ev[1].get() : nullptr);
        if (rc != LAMA_OK) { err_ = dm.error(); return rc; }
        return LAMA_OK;
    });
    if (rc != LAMA_OK) return rc;
    if (cells) *cells = bound[(size_t)n_clouds];
    if (counts) { counts[0] = events; counts[1] = pushes; }
    if (processed) std::copy(proc.begin(), proc.end(), processed);
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
    PS_TRY(cudaSetDevice(d.device));
    PS_TRY(d.record(0));
    PS_TRY(d.qin.reserve((size_t)n * 12));
    PS_TRY(d.ops.reserve((size_t)n));
    PS_TRY(d.changed.reserve((size_t)n));
    PS_TRY(d.ensure_records<uint32_t>((uint64_t)n));
    PS_TRY(cudaMemcpyAsync(d.qin.get(), cells_xyz, (size_t)n * 12, cudaMemcpyHostToDevice, d.stream));
    PS_TRY(cudaMemcpyAsync(d.ops.get(), ops, (size_t)n, cudaMemcpyHostToDevice, d.stream));
    PS_TRY(d.clear_marks());
    const uint32_t* xyz = (const uint32_t*)d.qin.get();
    const uint8_t* dops = (const uint8_t*)d.ops.get();
    const View v = d.view();
    k_om3_apply<false><<<blocks_for(n), kThreads, 0, d.stream>>>(xyz, dops, n, v, d.marks, d.status, nullptr, nullptr);
    d.launches[1] += 1;
    PS_TRY(cudaGetLastError());
    uint32_t status = 0;
    std::vector<uint32_t> marks;
    PS_TRY(d.read_marks(status, marks));
    if (status & kErrWindow) { err_ = "a cell lies outside the directory window"; return LAMA_ERR_WINDOW; }
    const int rc = d.alloc_marked(marks, v, err_, d.launches[1]);
    if (rc != LAMA_OK) return rc;
    k_om3_apply<true><<<blocks_for(n), kThreads, 0, d.stream>>>(xyz, dops, n, v, nullptr, nullptr, (uint32_t*)d.rk[0].get(), (uint32_t*)d.rv[0].get());
    PS_TRY(d.sort_fold<uint32_t, OpFold<true>>(n, v, d.kind, d.pp, (uint8_t*)d.changed.get()));
    d.launches[1] += 3;
    PS_TRY(cudaGetLastError());
    PS_TRY(d.record(1));
    if (changed) PS_TRY(cudaMemcpyAsync(changed, d.changed.get(), (size_t)n, cudaMemcpyDeviceToHost, d.stream));
    PS_TRY(d.finish(1));
    return LAMA_OK;
}

int OccMap3Dev::query(const uint32_t* cells_xyz, int n, double* prob, uint8_t* flags)
{
    Impl& d = *d_;
    if (n < 0 || (n > 0 && !cells_xyz)) { err_ = "null argument"; return LAMA_ERR_ARG; }
    if (n == 0) return LAMA_OK;
    PS_TRY(cudaSetDevice(d.device));
    PS_TRY(d.qin.reserve((size_t)n * 12));
    PS_TRY(d.qout.reserve((size_t)n * 4));
    PS_TRY(d.qflag.reserve((size_t)n));
    PS_TRY(cudaMemcpyAsync(d.qin.get(), cells_xyz, (size_t)n * 12, cudaMemcpyHostToDevice, d.stream));
    PS_TRY(d.record(0));
    k_om3_gather<<<blocks_for(n), kThreads, 0, d.stream>>>((const uint32_t*)d.qin.get(), n, d.view(), (uint32_t*)d.qout.get(), (uint8_t*)d.qflag.get());
    d.launches[2] += 1;
    PS_TRY(d.record(1));
    PS_TRY(cudaGetLastError());
    std::vector<uint32_t> words((size_t)n);
    std::vector<uint8_t> present((size_t)n);
    PS_TRY(cudaMemcpyAsync(words.data(), d.qout.get(), (size_t)n * 4, cudaMemcpyDeviceToHost, d.stream));
    PS_TRY(cudaMemcpyAsync(present.data(), d.qflag.get(), (size_t)n, cudaMemcpyDeviceToHost, d.stream));
    PS_TRY(d.finish(2));
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
    PS_TRY(cudaSetDevice(d.device));
    k_om3_prune<<<std::min<uint64_t>(8192, blocks_for((uint64_t)d.used << kOm3Log2Cells)), kThreads, 0, d.stream>>>(d.view(), d.used);
    PS_TRY(cudaGetLastError());
    PS_TRY(cudaStreamSynchronize(d.stream));
    return LAMA_OK;
}

int OccMap3Dev::bounds(uint32_t mn[3], uint32_t mx[3], int* patches) const
{
    d_->bounds(mn, mx, patches);
    return LAMA_OK;
}

int OccMap3Dev::export_box(const uint32_t lo[3], const int32_t size[3], uint32_t* words, uint8_t* known)
{
    void* const host[] = {words, known};
    return d_->export_box<BoxCell>(d_->view(), lo, size, host, err_);
}

// Map::write (map.cpp:490-529) with is_3d: patches in ascending directory index (the reference iterates an unordered_map)
int OccMap3Dev::write(const std::string& path)
{
    Impl& d = *d_;
    PS_TRY(cudaSetDevice(d.device));
    SdmFile f;
    const std::vector<int32_t> list = d.sdm_begin(f, 4, d.resolution);
    const View v = d.view();
    f.cells.resize(list.size() * (size_t)kOm3Cells * 4);
    f.masks.resize(list.size() * (size_t)kOm3Cells / 64);
    for (size_t j = 0; j < list.size(); ++j) {
        const int slot = d.h_dir[list[j]];
        PS_TRY(cudaMemcpyAsync(f.cells.data() + j * (size_t)kOm3Cells * 4, v.cells + ((size_t)slot << kOm3Log2Cells), (size_t)kOm3Cells * 4,
                               cudaMemcpyDeviceToHost, d.stream));
        // the mask words are 64-bit (container.cpp:39-43); two little-endian 32-bit known words make one
        PS_TRY(cudaMemcpyAsync(f.masks.data() + j * (size_t)kOm3Cells / 64, v.mask + (size_t)slot * kOm3KnownWords, (size_t)kOm3KnownWords * 4,
                               cudaMemcpyDeviceToHost, d.stream));
    }
    PS_TRY(cudaStreamSynchronize(d.stream));
    std::string err;
    if (!sdm_write(path, f, err)) { err_ = err; return LAMA_ERR_ARG; }
    return LAMA_OK;
}

// Map::read (map.cpp:531-575) into an empty map: the cell size and is_3d must match; the file's resolution is taken.  A patch the
// file holds twice is read twice: the last copy wins, as the reference's insert + read does.
int OccMap3Dev::read(const std::string& path)
{
    Impl& d = *d_;
    if (d.used != 0) { err_ = "read needs an empty map"; return LAMA_ERR_STATE; }
    SdmFile f;
    std::string err;
    if (!sdm_read(path, 4, 0, f, err, true)) { err_ = err; return LAMA_ERR_ARG; }
    std::vector<int> entry;
    int rc = d.sdm_entries(f, path, entry, err_);
    if (rc != LAMA_OK) return rc;
    std::vector<uint32_t> marks((size_t)d.ndir, 0);
    for (int di : entry) marks[di] = 1;
    PS_TRY(cudaSetDevice(d.device));
    const View v = d.view();
    rc = d.alloc_marked(marks, v, err_, d.launches[1]);
    if (rc != LAMA_OK) return rc;
    d.resolution = (double)f.header.resolution;   // map.cpp:548
    d.scale = 1.0 / d.resolution;
    for (size_t j = 0; j < f.ids.size(); ++j) {
        const int slot = d.h_dir[entry[j]];
        PS_TRY(cudaMemcpyAsync(v.cells + ((size_t)slot << kOm3Log2Cells), f.cells.data() + j * (size_t)kOm3Cells * 4, (size_t)kOm3Cells * 4,
                               cudaMemcpyHostToDevice, d.stream));
        PS_TRY(cudaMemcpyAsync(v.mask + (size_t)slot * kOm3KnownWords, f.masks.data() + j * (size_t)kOm3Cells / 64, (size_t)kOm3KnownWords * 4,
                               cudaMemcpyHostToDevice, d.stream));
    }
    PS_TRY(cudaStreamSynchronize(d.stream));
    return LAMA_OK;
}

// build_image (export.cpp:46-72) of the z-slice at w2m((0, 0, zed)).z, through the 2-D pixel rules of sdm_io.h
int OccMap3Dev::export_image(double zed, uint8_t* pixels, size_t cap, int dims[2])
{
    Impl& d = *d_;
    uint32_t lo[3];
    int32_t size[3];
    if (!d.image_box(zed, d.scale, pixels, cap, dims, lo, size)) return LAMA_OK;
    const size_t n = (size_t)size[0] * size[1];
    std::vector<uint32_t> words(n);
    std::vector<uint8_t> known(n);
    const int rc = export_box(lo, size, words.data(), known.data());
    if (rc != LAMA_OK) return rc;
    const SdmWindow win{lo[0], lo[1], size[0], size[1]};
    if (d.kind == kOm3Frequency) {
        std::vector<uint16_t> occupied(n), visited(n);
        for (size_t i = 0; i < n; ++i) {
            occupied[i] = (uint16_t)occ_occupied(words[i]);
            visited[i] = (uint16_t)occ_visited(words[i]);
        }
        sdm_occupancy_image_frequency(win, occupied.data(), visited.data(), known.data(), pixels);
    } else {
        std::vector<float> prob(n);
        for (size_t i = 0; i < n; ++i) prob[i] = om3_bits_float(words[i]);
        sdm_occupancy_image_logodds(win, prob.data(), known.data(), d.pp.thresh, pixels);
    }
    return LAMA_OK;
}

}  // namespace lama_b200
