// checkpoint.cpp -- PFSlam2D / Slam2D / GraphSlam2D checkpoints on the host (format: checkpoint.h, DESIGN.md §13): framing, checksum,
// every section once as a template over CkptWriter / CkptReader, and the save / load entry points of the handles.
#include "checkpoint.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <memory>
#include <sstream>

#include "frontend.h"

namespace lama_b200 {

int cuda_device_count();  // engine.cu

namespace {
using clk = std::chrono::steady_clock;
double ms_since(clk::time_point a) { return std::chrono::duration<double, std::milli>(clk::now() - a).count(); }
struct File {
    std::FILE* f;
    ~File() { if (f) std::fclose(f); }
};
}  // namespace

uint64_t fnv1a64(const uint8_t* p, size_t n, uint64_t h)
{
    for (size_t i = 0; i < n; ++i) {
        h ^= p[i];
        h *= 1099511628211ull;
    }
    return h;
}

int ckpt_write_file(const std::string& path, uint32_t kind, CkptWriter& w, const std::vector<CkptSegment>& tail, std::string& err, CheckpointStats* st)
{
    const auto t0 = std::chrono::steady_clock::now();
    if (w.version == kCkptVersionParked) {   // the marker opens the body, so that a reader of version 1 bodies cannot take it for one
        const uint8_t* m = reinterpret_cast<const uint8_t*>(&kCkptParkMarker);
        w.buf.insert(w.buf.begin() + kCkptHeaderBytes, m, m + 8);
    }
    uint8_t* h = w.buf.data();
    uint64_t total = (uint64_t)w.buf.size();
    uint64_t sum = fnv1a64(h + kCkptHeaderBytes, w.buf.size() - kCkptHeaderBytes);
    for (const CkptSegment& s : tail) {
        total += s.n;
        sum = fnv1a64(s.p, s.n, sum);
    }
    std::memcpy(h, &kCkptMagic, 8);
    std::memcpy(h + 8, &w.version, 4);
    std::memcpy(h + 12, &kind, 4);
    std::memcpy(h + 16, &total, 8);
    std::memcpy(h + 24, &sum, 8);
    const auto t1 = std::chrono::steady_clock::now();
    File f{std::fopen(path.c_str(), "wb")};
    if (!f.f) { err = "cannot open " + path + " for writing"; return LAMA_ERR_ARG; }
    bool ok = std::fwrite(w.buf.data(), 1, w.buf.size(), f.f) == w.buf.size();
    for (const CkptSegment& s : tail) ok = ok && (s.n == 0 || std::fwrite(s.p, 1, s.n, f.f) == s.n);
    if (!ok || std::fflush(f.f) != 0) {
        err = "write error on " + path;
        return LAMA_ERR_ARG;
    }
    std::fclose(f.f);
    f.f = nullptr;
    if (st) {
        st->encode_ms += std::chrono::duration<double, std::milli>(t1 - t0).count();
        st->io_ms += ms_since(t1);
        st->file_bytes = total;
    }
    return LAMA_OK;
}

int ckpt_read_file(const std::string& path, std::vector<uint8_t>& file, uint32_t* kind, std::string& err, CheckpointStats* st)
{
    const auto t0 = std::chrono::steady_clock::now();
    File f{std::fopen(path.c_str(), "rb")};
    if (!f.f) { err = "cannot open " + path; return LAMA_ERR_ARG; }
    if (std::fseek(f.f, 0, SEEK_END) != 0) { err = "cannot size " + path; return LAMA_ERR_ARG; }
    const long size = std::ftell(f.f);
    if (size < (long)kCkptHeaderBytes) { err = "not a checkpoint: shorter than its header"; return LAMA_ERR_ARG; }
    std::rewind(f.f);
    file.resize((size_t)size);
    if (std::fread(file.data(), 1, file.size(), f.f) != file.size()) { err = "read error on " + path; return LAMA_ERR_ARG; }
    const auto t1 = std::chrono::steady_clock::now();
    uint64_t magic, total, sum;
    uint32_t version;
    std::memcpy(&magic, file.data(), 8);
    std::memcpy(&version, file.data() + 8, 4);
    std::memcpy(kind, file.data() + 12, 4);
    std::memcpy(&total, file.data() + 16, 8);
    std::memcpy(&sum, file.data() + 24, 8);
    if (magic != kCkptMagic) { err = "not a checkpoint (bad magic)"; return LAMA_ERR_ARG; }
    uint64_t marker = 0;
    if (file.size() >= kCkptHeaderBytes + 8) std::memcpy(&marker, file.data() + kCkptHeaderBytes, 8);
    if (version != kCkptVersion && !(version == kCkptVersionParked && marker == kCkptParkMarker)) {
        err = "unsupported checkpoint format version " + std::to_string(version) + (version == kCkptVersionParked ? " (no parked-entry marker)" : "");
        return LAMA_ERR_ARG;
    }
    if (total != (uint64_t)file.size()) { err = "checkpoint size field differs from the file size (truncated or extended file)"; return LAMA_ERR_ARG; }
    if (fnv1a64(file.data() + kCkptHeaderBytes, file.size() - kCkptHeaderBytes) != sum) { err = "checkpoint checksum mismatch"; return LAMA_ERR_ARG; }
    if (st) {
        st->io_ms += std::chrono::duration<double, std::milli>(t1 - t0).count();
        st->encode_ms += ms_since(t1);
        st->file_bytes = file.size();
    }
    return LAMA_OK;
}

CkptReader ckpt_body(const std::vector<uint8_t>& file)
{
    uint32_t version = kCkptVersion;
    std::memcpy(&version, file.data() + 8, 4);
    const size_t skip = kCkptHeaderBytes + (version == kCkptVersionParked ? 8 : 0);
    return CkptReader(file.data() + skip, file.size() - skip, version);
}

namespace {
// the fixed fields of an engine section (Img: EngineImage, const for the writer)
template <class IO, class Img> void engine_fields(IO& io, Img& img)
{
    io.i32(img.particles, "particles"); io.i32(img.dir_dim, "dir_dim"); io.i32(img.pool_slots, "pool_slots"); io.i32(img.max_beams, "max_beams");
    io.i32(img.occupancy_kind, "occupancy kind");
    io.u8(img.known_plane, "known plane");
    io.f64(img.resolution, "resolution"); io.f64(img.l2_max, "l2_max");
    io.i32(img.window.base_px, "window"); io.i32(img.window.base_py, "window");
    for (auto& c : img.counters) io.u64(c, "store counters");
    io.u32(img.used, "used slots");
}
}  // namespace

void ckpt_put_engine(CkptWriter& w, const EngineImage* img)
{
    if (img && !img->parked.empty()) w.version = kCkptVersionParked;
    w.u8(img != nullptr);
    if (!img) return;
    engine_fields(w, *img);
    w.array(img->refcount, img->refcount.size(), nullptr);
    w.array(img->dirs, img->dirs.size(), nullptr);
    if (w.version == kCkptVersionParked) {
        const size_t n_lists = (size_t)img->particles * img->n_kinds();
        for (size_t li = 0; li < n_lists; ++li) w.u32(li < img->park_len.size() ? (uint32_t)img->park_len[li] : 0u);
        for (const ParkEntry& e : img->parked) { w.i32(e.px); w.i32(e.py); w.i32(e.entry); }
    }
}

bool ckpt_get_engine(CkptReader& r, bool* present, EngineImage& img, int particles, int occupancy_kind, bool last)
{
    r.u8(*present, "engine flag");
    if (!r.ok() || !*present) return r.ok();
    engine_fields(r, img);
    img.window.dim = img.dir_dim;
    if (!r.ok()) return false;
    if (img.particles < 1 || (particles >= 0 && img.particles != particles)) { r.fail("engine particle count differs from the front end's"); return false; }
    if (img.dir_dim < 8 || img.dir_dim > 128 || (img.dir_dim & (img.dir_dim - 1)) != 0) { r.fail("bad dir_dim"); return false; }
    if (img.pool_slots < 1 || img.pool_slots >= kDirSlotMask) { r.fail("bad pool size"); return false; }
    if (img.max_beams < 1 || img.max_beams > 32768) { r.fail("bad max_beams"); return false; }
    if (img.occupancy_kind < 0 || img.occupancy_kind > 1 || (occupancy_kind >= 0 && img.occupancy_kind != occupancy_kind)) { r.fail("bad occupancy kind"); return false; }
    if (!(img.resolution > 0) || !(img.l2_max >= 0) || std::ceil(img.l2_max / img.resolution) > 63.0) { r.fail("bad resolution / l2_max"); return false; }
    const int64_t max_patch = (int64_t)1 << (32 - kPatchLog2);
    if (img.window.base_px < 0 || img.window.base_py < 0 || img.window.base_px + img.dir_dim > max_patch || img.window.base_py + img.dir_dim > max_patch) {
        r.fail("directory window outside the map");
        return false;
    }
    if (img.used > (uint32_t)img.pool_slots) { r.fail("more used slots than pool slots"); return false; }
    const uint64_t n_dir = (uint64_t)img.particles * img.n_kinds() * img.dir_dim * img.dir_dim;
    // every count against the bytes that are left, before anything is allocated
    uint64_t need = (uint64_t)img.used * 4 + n_dir * 4 + (uint64_t)img.used * img.slot_stride();
    if (need > r.left()) { r.fail("engine section exceeds the file"); return false; }
    r.array(img.refcount, img.used, "reference counts");
    r.array(img.dirs, n_dir, "directories");
    img.park_len.clear();
    img.parked.clear();
    if (r.version == kCkptVersionParked) {   // the parked lists
        const size_t n_lists = (size_t)img.particles * img.n_kinds();
        r.array(img.park_len, n_lists, "parked list lengths");
        uint64_t total = 0;
        for (int32_t n : img.park_len) {
            if (n < 0) { r.fail("negative parked list length"); return false; }
            total += (uint64_t)n;
        }
        r.count(total, 12, "parked entries");
        std::vector<int32_t> raw;
        r.array(raw, (size_t)total * 3, "parked entries");
        if (!r.ok()) return false;
        img.parked.resize((size_t)total);
        for (size_t i = 0; i < img.parked.size(); ++i) img.parked[i] = ParkEntry{raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]};
        size_t at = 0;
        for (int32_t n : img.park_len) {
            for (int32_t k = 0; k < n; ++k, ++at) {
                const ParkEntry& e = img.parked[at];
                if (k > 0 && !park_before(img.parked[at - 1].px, img.parked[at - 1].py, e.px, e.py)) { r.fail("parked list not strictly sorted"); return false; }
                if (e.px < 0 || e.py < 0 || e.px >= max_patch || e.py >= max_patch || patch_in_window(img.window, e.px, e.py)) {
                    r.fail("parked entry inside the saved window or outside the map");
                    return false;
                }
            }
        }
        if (total == 0) img.park_len.clear();
    }
    need = (uint64_t)img.used * img.slot_stride();
    if (need > r.left() || (last && need != r.left())) { r.fail(need > r.left() ? "engine section exceeds the file" : "bytes after the engine section"); return false; }
    img.slot_bytes = r.take((size_t)img.used * img.slot_stride(), "slots");
    if (!r.ok()) return false;
    std::vector<int32_t> refs(img.used, 0);
    constexpr int32_t flags = kDirHot | kDirOwn;
    for (int32_t e : img.dirs) {
        if (e == -1) continue;
        if (e < 0 || (e & ~(kDirSlotMask | flags)) != 0) { r.fail("directory entry with unknown flag bits"); return false; }
        const uint32_t slot = (uint32_t)(e & kDirSlotMask);
        if (slot >= img.used) { r.fail("directory entry points past the saved slots"); return false; }
        ++refs[slot];
    }
    for (const ParkEntry& p : img.parked) {
        const int32_t e = p.entry;
        if (e < 0 || (e & ~(kDirSlotMask | flags)) != 0) { r.fail("parked entry with unknown flag bits"); return false; }
        const uint32_t slot = (uint32_t)(e & kDirSlotMask);
        if (slot >= img.used) { r.fail("parked entry points past the saved slots"); return false; }
        ++refs[slot];
    }
    for (uint32_t s = 0; s < img.used; ++s)
        if (refs[s] != img.refcount[s]) { r.fail("reference count differs from the directory references of slot " + std::to_string(s)); return false; }
    return true;
}

bool ckpt_check_rng(const std::string& text)
{
    std::istringstream in(text);
    unsigned long long v = 0;
    int n = 0;
    while (in >> v) {
        if (v > 0xFFFFFFFFull) return false;
        ++n;
        if (n == 625 && v > 624) return false;
    }
    return in.eof() && n == 625;
}

namespace {
bool finite_se2(const SE2& s) { return std::isfinite(s.c) && std::isfinite(s.s) && std::isfinite(s.tx) && std::isfinite(s.ty); }
bool finite(const double* v, int n)
{
    for (int k = 0; k < n; ++k)
        if (!std::isfinite(v[k])) return false;
    return true;
}
uint64_t sum_refs(const EngineImage& img)
{
    uint64_t n = 0;
    for (int32_t v : img.refcount) n += (uint64_t)v;
    return n;
}
void add_times(CheckpointTimes& a, const CheckpointTimes& b)
{
    a.count_ms += b.count_ms; a.compact_ms += b.compact_ms; a.gather_ms += b.gather_ms;
    a.copy_ms += b.copy_ms; a.create_ms += b.create_ms; a.tables_ms += b.tables_ms;
}
// the refusal of a loader called on another handle kind's file
std::string wrong_kind(uint32_t kind, const char* want)
{
    const char* held = kind == kCkptPFSlam2D ? "PFSlam2D"
                       : kind == kCkptPFSlam2DShard ? "PFSlam2D shard"
                       : kind == kCkptSlam2D || kind == kCkptLidarOdometry2D ? "Slam2D"
                       : kind == kCkptGraphSlam2D ? "GraphSlam2D" : nullptr;
    return held ? std::string("the checkpoint holds a ") + held + ", not a " + want : std::string("unknown checkpoint handle kind");
}
// the caller's dir_dim / pool_slots / max_beams: 0, or the file's (its options, or the engine it holds)
bool geometry_matches(const DeviceOptions& call, const DeviceOptions& file, const EngineImage* img, std::string& err)
{
    auto ok = [](int v, int opt, int eng) { return v == 0 || v == opt || v == eng; };
    if (ok(call.dir_dim, file.dir_dim, img ? img->dir_dim : file.dir_dim) && ok(call.pool_slots, file.pool_slots, img ? img->pool_slots : file.pool_slots) &&
        ok(call.max_beams, file.max_beams, img ? img->max_beams : file.max_beams))
        return true;
    err = "device options differ from the checkpoint's geometry (dir_dim, pool_slots and max_beams must be 0 or the saved values)";
    return false;
}
bool same_engine_geometry(const EngineImage& a, const EngineImage& b)
{
    return a.dir_dim == b.dir_dim && a.pool_slots == b.pool_slots && a.max_beams == b.max_beams && a.occupancy_kind == b.occupancy_kind &&
           a.known_plane == b.known_plane && a.resolution == b.resolution && a.l2_max == b.l2_max;
}
// the session id of a shard file: FNV-1a-64 of its options and state sections without the rank-local fields (offsets from `body`)
uint64_t session_id(const uint8_t* body, size_t shared, const size_t marks[3], size_t end)
{
    return fnv1a64(body + marks[2], end - marks[2], fnv1a64(body + shared, marks[1] - shared));
}

// What every save shares: fresh statistics, the snapshots of the handle's engines, the clocks, and the file -- the sections the caller
// writes into w, then each engine section followed by its slots.
class SaveFrame {
public:
    explicit SaveFrame(CheckpointStats* st) : s(st ? *st : local_) { s = CheckpointStats(); imgs_.reserve(2); }
    CheckpointStats& s;
    CkptWriter w;
    // the next engine section: a snapshot of e's first `particles` (0: all), or an absent section when e is null
    int snapshot(Engine* e, std::string& err, int particles = 0)
    {
        imgs_.emplace_back();
        present_.push_back(e != nullptr);
        if (e) {
            CheckpointTimes t;
            const int rc = e->snapshot(&imgs_.back(), &t, particles);
            if (rc != LAMA_OK) { err = e->last_error(); return rc; }
            add_times(s.dev, t);
        }
        t1_ = clk::now();
        return LAMA_OK;
    }
    int write(const std::string& path, uint32_t kind, std::string& err)
    {
        std::vector<CkptWriter> more(imgs_.size());   // the engine sections after the first: own buffers, framed like the first
        std::vector<CkptSegment> tail;
        uint64_t used = 0, refs = 0;
        // one version for the whole file: every engine section carries parked lists when any of them has parked entries (a GraphSlam2D
        // whose global map has moved and whose inner map has not)
        for (size_t i = 0; i < imgs_.size(); ++i)
            if (present_[i] && !imgs_[i].parked.empty()) w.version = kCkptVersionParked;
        for (size_t i = 0; i < imgs_.size(); ++i) {
            const EngineImage& img = imgs_[i];
            CkptWriter& to = i == 0 ? w : more[i];
            if (i > 0) { to.buf.clear(); to.version = w.version; }
            ckpt_put_engine(to, present_[i] ? &img : nullptr);
            if (i > 0) tail.push_back({to.buf.data(), to.buf.size()});
            tail.push_back({img.slot_bytes, (size_t)img.used * img.slot_stride()});
            used += img.used;
            refs += sum_refs(img);
        }
        s.encode_ms = ms_since(t1_);
        const int rc = ckpt_write_file(path, kind, w, tail, err, &s);
        if (rc != LAMA_OK) return rc;
        s.used_slots = used;
        s.references = refs;
        s.total_ms   = ms_since(t0_);
        return LAMA_OK;
    }

private:
    CheckpointStats local_;
    clk::time_point t0_ = clk::now(), t1_ = t0_;
    std::vector<EngineImage> imgs_;
    std::vector<bool> present_;
};

// What every load shares: fresh statistics, *code (LAMA_ERR_ARG until done), the file reads, the parse clock, the refusal without a
// device and the engine restores.
class LoadFrame {
public:
    LoadFrame(CheckpointStats* st, int* code, std::string& err) : s(st ? *st : local_), code_(code), err_(err)
    {
        s = CheckpointStats();
        *code = LAMA_ERR_ARG;
    }
    CheckpointStats& s;
    // reads `path` and checks its header; the parse clock starts
    bool read(const std::string& path, std::vector<uint8_t>& file, uint32_t* kind)
    {
        *code_ = ckpt_read_file(path, file, kind, err_, &s);
        if (*code_ != LAMA_OK) return false;
        *code_ = LAMA_ERR_ARG;
        bytes_ += file.size();
        t1_ = clk::now();
        return true;
    }
    // the end of a file's sections: nothing may follow them
    bool checked(CkptReader& r)
    {
        r.check(r.left() != 0, "bytes after the last section");
        if (!r.ok()) err_ = r.error();
        return r.ok();
    }
    void parsed() { s.encode_ms += ms_since(t1_); }
    // the file is valid: from here on the device
    bool device()
    {
        if (cuda_device_count() >= 1) return true;
        *code_ = LAMA_ERR_NO_DEVICE;
        err_ = "no CUDA device available: the lama_b200 hot path has no CPU fallback";
        return false;
    }
    Engine* restore(const EngineImage& img, const DeviceOptions& dev, int capacity = 0)
    {
        CheckpointTimes t;
        Engine* e = Engine::restore(img, dev.device, dev.stream, err_, &t, capacity);
        if (!e) { *code_ = LAMA_ERR_CUDA; return nullptr; }
        e->enable_timing(dev.timing != 0);
        add_times(s.dev, t);
        used_ += img.used;
        refs_ += sum_refs(img);
        return e;
    }
    template <class T> T* done(std::unique_ptr<T>& p)
    {
        s.used_slots = used_;
        s.references = refs_;
        s.file_bytes = bytes_;
        s.total_ms   = ms_since(t0_);
        *code_ = LAMA_OK;
        return p.release();
    }

private:
    CheckpointStats local_;
    int* code_;
    std::string& err_;
    clk::time_point t0_ = clk::now(), t1_ = t0_;
    uint64_t bytes_ = 0, used_ = 0, refs_ = 0;
};
}  // namespace

// The sections, each once for both directions, and the loaders' assembly; a friend of the handles.
struct Ckpt {
    template <class IO> static void counters(IO& io, Counters& c)
    {
        for (uint64_t* v : {&c.evals, &c.ray_cells, &c.dm_pops, &c.detached, &c.gn_iters, &c.resampled}) io.u64(*v, "counters");
    }
    template <class IO> static void geometry(IO& io, DeviceOptions& d)
    {
        io.i32(d.dir_dim, "dir_dim"); io.i32(d.pool_slots, "pool_slots"); io.i32(d.max_beams, "max_beams");
    }

    // ---- PFSlam2D (kinds 1 and 5) ----
    // The options and state sections.  marks = {end of the options, start and end of the rank-local fields}, as offsets into w.buf /
    // from the reader's start.
    template <class IO> static void pf_sections(IO& io, PFSlam2D& h, size_t marks[3])
    {
        PFOptions& o = h.opt_;
        io.u32(o.particles, "options");
        for (double* v : {&o.srr, &o.str, &o.stt, &o.srt, &o.meas_sigma, &o.meas_sigma_gain, &o.trans_thresh, &o.rot_thresh, &o.l2_max, &o.truncated_ray,
                          &o.truncated_range, &o.resolution})
            io.f64(*v, "options");
        io.u32(o.patch_size, "options"); io.u32(o.max_iter, "options"); io.i32(o.strategy, "options"); io.i32(o.threads, "options"); io.u32(o.seed, "options");
        geometry(io, o.dev);
        io.check(o.particles < 1 || o.patch_size != 32 || !(o.resolution > 0) || o.dev.dir_dim < 8 || o.dev.max_beams < 1 || o.dev.pool_slots < 0, "bad options");
        marks[0] = io.pos();
        const uint32_t P = io.ok() ? o.particles : 0;
        // front-end state
        io.se2(h.prior_, "state"); io.se2(h.odom_, "state"); io.u8(h.has_first_, "state");
        io.f64(h.acc_trans_, "state"); io.f64(h.acc_rot_, "state"); io.f64(h.neff_, "state");
        io.array(h.pose_, P, "poses");
        io.array(h.weight_, P, "weights"); io.array(h.nweight_, P, "weights"); io.array(h.wsum_, P, "weights");
        io.vec(h.last_idx_, "resample indices");
        io.u64(h.resample_count_, "resample digest"); io.u64(h.resample_hash_, "resample digest"); io.u64(h.scans_seen_, "resample digest");
        io.vec(h.timestamps_, "timestamps");
        marks[1] = io.pos();
        rank_local(io, h);
        marks[2] = io.pos();
        // the trajectory nodes reachable from the particles, renumbered in their old order (a parent precedes its children)
        if constexpr (!IO::kLoad) {
            std::vector<int> renum(h.nodes_.size(), -1);
            for (uint32_t i = 0; i < P; ++i)
                for (int n = h.node_of_[i]; n >= 0 && renum[(size_t)n] < 0; n = h.nodes_[(size_t)n].parent) renum[(size_t)n] = 0;
            uint32_t kept = 0;
            for (int& v : renum)
                if (v == 0) v = (int)kept++;
            io.u32(kept);
            for (size_t n = 0; n < h.nodes_.size(); ++n)
                if (renum[n] >= 0) {
                    io.se2(h.nodes_[n].pose);
                    io.i32(h.nodes_[n].parent < 0 ? -1 : renum[(size_t)h.nodes_[n].parent]);
                }
            for (uint32_t i = 0; i < P; ++i) io.i32(h.node_of_[i] < 0 ? -1 : renum[(size_t)h.node_of_[i]]);
        } else {
            io.length(h.nodes_, 4 * 8 + 4, "nodes");
            for (size_t n = 0; n < h.nodes_.size(); ++n) {
                io.se2(h.nodes_[n].pose, "nodes");
                io.i32(h.nodes_[n].parent, "nodes");
                io.check(h.nodes_[n].parent < -1 || h.nodes_[n].parent >= (int)n, "a trajectory node does not follow its parent");
            }
            io.array(h.node_of_, P, "trajectory heads");
        }
        std::string rng;
        if constexpr (!IO::kLoad) {
            std::ostringstream out;
            out << h.gen_;
            rng = out.str();
        }
        io.str(rng, "random generator");
        if constexpr (IO::kLoad) {
            for (int32_t v : h.last_idx_) io.check(v < 0 || v >= (int32_t)P, "resample index out of range");
            io.check(!h.last_idx_.empty() && h.last_idx_.size() != P, "resample indices of the wrong length");
            for (int32_t v : h.node_of_) io.check(v < -1 || v >= (int32_t)h.nodes_.size() || (h.has_first_ && v < 0), "trajectory head out of range");
            io.check(!ckpt_check_rng(rng), "malformed random generator state");
            io.check(!finite_se2(h.prior_) || !finite_se2(h.odom_), "non-finite pose");
            if (io.ok()) {
                std::istringstream in(rng);
                in >> h.gen_;
            }
        }
    }
    // the fields each rank of one filter holds for itself (a shard file's session id skips them)
    template <class IO> static void rank_local(IO& io, PFSlam2D& h)
    {
        counters(io, h.last_); counters(io, h.total_);
        io.u64(h.detached_seen_, "counters");
        for (double* v : {&h.t_sample_, &h.t_solve_, &h.t_norm_, &h.t_resample_}) io.f64(*v, "summary");
    }
    static void copy_rank_local(PFSlam2D& to, const PFSlam2D& from)
    {
        to.last_ = from.last_; to.total_ = from.total_; to.detached_seen_ = from.detached_seen_;
        to.t_sample_ = from.t_sample_; to.t_solve_ = from.t_solve_; to.t_norm_ = from.t_norm_; to.t_resample_ = from.t_resample_;
    }

    static int save_pf(PFSlam2D& h, const std::string& path, bool shard, SaveFrame& f)
    {
        if (h.eng_) {
            const int rc = h.settle_counters();   // the pending map update and its counters, as the getters would book them
            if (rc != LAMA_OK) return rc;
        }
        int rc = f.snapshot(h.eng_.get(), h.err_, h.hi_ - h.lo_);   // the local particles; a sharded engine's staging particles are not saved
        if (rc != LAMA_OK) return rc;
        CkptWriter& w = f.w;
        size_t id_at = 0;
        if (shard) {
            w.u32(h.opt_.shard_rank); w.u32(h.opt_.shard_count);
            id_at = w.pos();
            w.u64(0);
        }
        const size_t shared = w.pos();
        size_t marks[3];
        pf_sections(w, h, marks);
        if (shard) {
            const uint64_t id = session_id(w.buf.data(), shared, marks, w.pos());
            std::memcpy(w.buf.data() + id_at, &id, 8);
        }
        return f.write(path, shard ? kCkptPFSlam2DShard : kCkptPFSlam2D, h.err_);
    }

    // One file of a kind-1 file or a kind-5 set, read and checked, and what it gives the new rank: its kept slots (ascending old ids)
    // and the directories of the particles it gives.
    struct ShardSource {
        std::vector<uint8_t> file;               // the whole file, kept when every slot is needed
        uint32_t rank = 0, count = 1;
        uint64_t id = 0;
        std::unique_ptr<PFSlam2D> h;             // the options and state sections, on a handle without a device
        std::vector<uint8_t> options;            // the options section, byte for byte
        EngineImage img;
        bool has_engine = false;
        std::vector<uint32_t> kept;              // old slot ids
        std::vector<int32_t> remap;              // old slot -> position in `kept` (-1: not kept)
        std::vector<int32_t> dirs;               // the directories of the particles this file gives, in global particle order
        std::vector<uint8_t> slots;              // when not every slot is kept: the kept slots only, as a payload of kept.size() slots
        const uint8_t* payload = nullptr;
        uint32_t payload_count = 0;
    };
    static bool read_source(LoadFrame& f, const std::string& path, bool whole_only, bool several, ShardSource& so, std::string& err)
    {
        uint32_t kind = 0;
        if (!f.read(path, so.file, &kind)) return false;
        if (kind == kCkptPFSlam2DShard && whole_only) {
            err = "the checkpoint holds one shard of a sharded PFSlam2D: load the complete set of shard files with lama_pf_load_state_sharded";
            return false;
        }
        if (kind != kCkptPFSlam2D && kind != kCkptPFSlam2DShard) { err = wrong_kind(kind, "PFSlam2D"); return false; }
        if (kind == kCkptPFSlam2D && several) { err = "a whole-filter checkpoint (kind 1) cannot be mixed with other files: load it alone"; return false; }
        CkptReader r = ckpt_body(so.file);
        if (kind == kCkptPFSlam2DShard) {
            r.u32(so.rank, "shard record"); r.u32(so.count, "shard record"); r.u64(so.id, "shard record");
            r.check(so.count < 2 || so.rank >= so.count, "bad shard record (shard_rank must be below shard_count >= 2)");
        }
        const size_t shared = r.pos();
        size_t marks[3];
        so.h.reset(new PFSlam2D());
        pf_sections(r, *so.h, marks);
        const uint32_t P = r.ok() ? so.h->opt_.particles : 0;
        r.check(P % so.count != 0, "the particles do not divide evenly over the file's shard count");
        const uint8_t* body = so.file.data() + kCkptHeaderBytes;
        if (r.ok() && kind == kCkptPFSlam2DShard) r.check(session_id(body, shared, marks, r.pos()) != so.id, "session id differs from the file's shared sections");
        if (r.ok()) ckpt_get_engine(r, &so.has_engine, so.img, (int)(P / so.count), 0);
        r.check(!so.img.parked.empty() && !whole_only,
                "the session's maps have parked entries (its window moved with the robot); sharded sessions keep a fixed window, load it with lama_pf_load_state");
        r.check(so.h->has_first_ && !so.has_engine, "a filter past its first scan without device state");
        if (!f.checked(r)) return false;
        so.options.assign(body + shared, body + marks[0]);
        return true;
    }
    // a later file of a set against the first
    static bool same_set(const ShardSource& a, const ShardSource& first, std::string& err)
    {
        if (a.count != first.count) { err = "the shard files disagree about the shard count"; return false; }
        if (a.options != first.options) { err = "the shard files hold different options"; return false; }
        if (a.has_engine != first.has_engine || (first.has_engine && !same_engine_geometry(a.img, first.img))) {
            err = "the shard files hold different engine geometry";
            return false;
        }
        if (first.has_engine && (a.img.window.base_px != first.img.window.base_px || a.img.window.base_py != first.img.window.base_py)) {
            err = "the shard files hold different directory windows";
            return false;
        }
        if (a.id != first.id) { err = "the shard files come from different saves (session ids differ)"; return false; }
        return true;
    }
    // keeps what `so` gives the new rank's particles, global [lo, lo + per): their directories and parked lists and the slots they
    // reference; the rest of the file is dropped
    static void take_particles(ShardSource& so, uint32_t lo, uint32_t per)
    {
        EngineImage& img = so.img;
        const uint32_t per_src = (uint32_t)img.particles, a = std::max(lo, so.rank * per_src), b = std::min(lo + per, (so.rank + 1) * per_src);
        if (!so.has_engine || a >= b) {
            img.parked.clear();
        } else {
            const size_t dir_n = (size_t)img.n_kinds() * img.dir_dim * img.dir_dim;
            so.dirs.assign(img.dirs.begin() + (size_t)(a - so.rank * per_src) * dir_n, img.dirs.begin() + (size_t)(b - so.rank * per_src) * dir_n);
            so.remap.assign(img.used, -1);
            for (int32_t e : so.dirs)
                if (e != -1) so.remap[(size_t)(e & kDirSlotMask)] = 0;
            for (const ParkEntry& pe : img.parked) so.remap[(size_t)(pe.entry & kDirSlotMask)] = 0;   // whole-session files only
            for (uint32_t k = 0; k < img.used; ++k)
                if (so.remap[k] == 0) { so.remap[k] = (int32_t)so.kept.size(); so.kept.push_back(k); }
            const size_t stride = img.slot_stride(), n = so.kept.size();
            if (n == img.used) {   // every slot: keep the file instead of copying its slots
                so.payload_count = img.used;
                so.payload = img.slot_bytes;
                return;
            }
            // only the kept slots, as a payload of n slots: cells, then mirror bits, then known bits
            so.slots.resize(n * stride);
            const size_t planes[3] = {0, (size_t)img.used * kPatchBytes, (size_t)img.used * (kPatchBytes + 128)};
            const size_t pieces[3] = {(size_t)kPatchBytes, 128, 128}, out[3] = {0, n * kPatchBytes, n * (kPatchBytes + 128)};
            for (int p = 0; p < (img.has_kbits() ? 3 : 2); ++p)
                for (size_t j = 0; j < n; ++j)
                    std::memcpy(so.slots.data() + out[p] + j * pieces[p], img.slot_bytes + planes[p] + (size_t)so.kept[j] * pieces[p], pieces[p]);
            so.payload = so.slots.data();
            so.payload_count = (uint32_t)n;
        }
        img.slot_bytes = nullptr;
        std::vector<uint8_t>().swap(so.file);
    }
    // The engine image of the new rank over `img`'s geometry, window and counters: kept slots numbered in ascending (source rank, old
    // slot) order, directories and parked lists remapped, reference counts recounted.
    static bool assemble(const std::vector<ShardSource>& src, EngineImage& img, std::string& err)
    {
        std::vector<uint32_t> base(src.size(), 0);
        uint32_t K = 0;
        for (size_t k = 0; k < src.size(); ++k) {
            base[k] = K;
            K += (uint32_t)src[k].kept.size();
        }
        if (img.pool_slots >= (int)kDirSlotMask || K > (uint32_t)img.pool_slots) {
            err = "the " + std::to_string(K) + " slots this rank keeps do not fit a pool of " + std::to_string(img.pool_slots) + " slots (raise pool_slots)";
            return false;
        }
        img.used = K;
        img.refcount.assign(K, 0);
        img.dirs.clear();
        img.dirs.reserve((size_t)img.particles * img.n_kinds() * img.dir_dim * img.dir_dim);
        img.park_len.clear();
        img.parked.clear();
        img.slot_bytes = nullptr;
        img.slot_src.resize(K);
        for (size_t k = 0; k < src.size(); ++k) {
            const ShardSource& so = src[k];
            for (int32_t e : so.dirs) {
                if (e == -1) { img.dirs.push_back(-1); continue; }
                const uint32_t id = base[k] + (uint32_t)so.remap[(size_t)(e & kDirSlotMask)];
                ++img.refcount[id];
                img.dirs.push_back((int32_t)id | (e & ~kDirSlotMask));
            }
            if (!so.img.parked.empty()) img.park_len = so.img.park_len;
            for (const ParkEntry& pe : so.img.parked) {
                const uint32_t id = base[k] + (uint32_t)so.remap[(size_t)(pe.entry & kDirSlotMask)];
                ++img.refcount[id];
                img.parked.push_back(ParkEntry{pe.px, pe.py, (int32_t)id | (pe.entry & ~kDirSlotMask)});
            }
            for (size_t j = 0; j < so.kept.size(); ++j)
                img.slot_src[base[k] + j] = EngineImage::SlotRef{so.payload, so.payload_count, so.payload == so.slots.data() ? (uint32_t)j : so.kept[j]};
            if (K > 0 && so.kept.size() == K && so.payload_count == K) {   // one file gives every slot, in its own order: one contiguous copy
                img.slot_bytes = so.payload;
                img.slot_src.clear();
            }
        }
        return true;
    }

    // ---- Slam2D (kinds 2 and 3, and the inner Slam2D of kind 4) ----
    // the options and state sections; lidar_odometry: what the file kind says (the reader checks it)
    template <class IO> static void slam_sections(IO& io, Slam2D& h, bool lidar_odometry)
    {
        SlamOptions& o = h.opt_;
        for (double* v : {&o.trans_thresh, &o.rot_thresh, &o.l2_max, &o.truncated_ray, &o.truncated_range, &o.resolution}) io.f64(*v, "options");
        io.u32(o.patch_size, "options"); io.u32(o.max_iter, "options"); io.i32(o.strategy, "options"); io.i32(o.occupancy, "options");
        io.u8(o.transient_map, "options"); io.u8(o.lidar_odometry, "options");
        geometry(io, o.dev);
        io.check(o.patch_size != 32 || !(o.resolution > 0) || o.occupancy < 0 || o.occupancy > 1 || o.dev.dir_dim < 8 || o.dev.max_beams < 1 ||
                     o.dev.pool_slots < 0 || o.lidar_odometry != lidar_odometry,
                 "bad options");
        io.se2(h.pose_, "state"); io.se2(h.odom_, "state"); io.se2(h.map_update_pose_, "state");
        io.u8(h.has_first_, "state"); io.u8(h.engine_ready_, "state");
        io.u32(h.processed_, "state"); io.u64(h.removed_, "state"); io.u64(h.map_updates_, "state");
        counters(io, h.last_); counters(io, h.total_);
        io.check(!finite_se2(h.pose_) || !finite_se2(h.odom_) || !finite_se2(h.map_update_pose_), "non-finite pose");
    }
    // a checked Slam2D on dev.device / dev.stream with dev.timing: the checks create() applies, then its engine from `img` (null: none)
    static bool restore_slam(LoadFrame& f, Slam2D& s, const EngineImage* img, const DeviceOptions& dev, std::string& err)
    {
        s.opt_.dev.device = dev.device; s.opt_.dev.stream = dev.stream; s.opt_.dev.timing = dev.timing;
        if (!Slam2D::valid_options(s.opt_, err) || !f.device()) return false;
        if (img) {
            s.eng_.reset(f.restore(*img, dev));
            if (!s.eng_) return false;
            s.eng_->set_lidar_odometry_rays(s.opt_.lidar_odometry);
        }
        return true;
    }

    // ---- GraphSlam2D (kind 4) ----
    template <class IO> static void loss(IO& io, PgoLoss& l, const char* what)
    {
        for (double& v : l.sigma) io.f64(v, what);
        io.f64(l.huber_k, what);
        bool ok = l.huber_k >= 0 && std::isfinite(l.huber_k);
        for (double v : l.sigma) ok = ok && v > 0 && std::isfinite(v);   // GraphSlam2D's sigmas are finite constants; inf would drop a factor
        io.check(!ok, "bad loss", what);
    }
    template <class IO> static void betweens(IO& io, std::vector<PgoBetween>& v, size_t n_keys, const char* what)
    {
        io.length(v, 2 * 4 + 4 * 8 + 4 * 8, what);
        for (PgoBetween& b : v) {
            io.i32(b.from, what); io.i32(b.to, what); io.se2(b.measured, what);
            loss(io, b.loss, what);
            io.check(b.from < 0 || (size_t)b.from >= n_keys || b.to < 0 || (size_t)b.to >= n_keys, "a factor names no key", what);
            io.check(!finite_se2(b.measured), "non-finite factor", what);
        }
    }
    // every section before the engines; center: the inner Slam2D's window centre (a restored engine does not know it, Engine::set_center)
    template <class IO> static void graph_sections(IO& io, GraphSlam2D& g, double center[2])
    {
        GraphOptions& o = g.opt_;
        io.f64(o.key_pose_distance, "graph options"); io.f64(o.key_pose_angular_distance, "graph options"); io.i32(o.key_pose_head_delay, "graph options");
        io.f64(o.loop_search_max_distance, "graph options"); io.f64(o.loop_search_min_distance, "graph options"); io.i32(o.loop_max_candidates, "graph options");
        io.f64(o.loop_closure_scan_rmse, "graph options"); io.i32(o.loop_closure_max_candidates, "graph options"); io.i32(o.ignore_n_chain_poses, "graph options");
        // an infinite threshold is a user's way to switch a test off (key_pose_angular_distance = inf: keys by distance only), so only NaN is refused
        bool nan = false;
        for (double v : {o.key_pose_distance, o.key_pose_angular_distance, o.loop_search_max_distance, o.loop_search_min_distance, o.loop_closure_scan_rmse})
            nan = nan || std::isnan(v);
        io.check(nan || o.key_pose_head_delay < 0 || o.ignore_n_chain_poses < 0 || o.loop_max_candidates < 0, "bad graph options");
        // the inner Slam2D: the bytes of a kind-2 file's options and state
        Slam2D& s = *g.slam_;
        slam_sections(io, s, false);
        io.check(!s.opt_.transient_map || s.opt_.truncated_ray != 1.0 || s.opt_.occupancy != 0,
                 "the inner Slam2D's options are not the ones GraphSlam2D forces (transient map, truncated_ray 1, frequency map, no lidar odometry)");
        // graph state
        io.se2(g.correction_, "graph state"); io.se2(g.prev_, "graph state");
        io.f64(g.accdist_, "graph state"); io.f64(g.factordist_, "graph state");
        io.u64(g.mapping_keyid_, "graph state");
        io.u64(g.stats_.loop_factors, "graph stats"); io.u64(g.stats_.optimizations, "graph stats"); io.u64(g.stats_.optimizations_ok, "graph stats");
        PgoReport& rep = g.stats_.last;
        io.i32(rep.status, "last report"); io.u32(rep.iterations, "last report"); io.u32(rep.lambda_tries, "last report"); io.u64(rep.cg_iterations, "last report");
        io.f64(rep.initial_error, "last report"); io.f64(rep.final_error, "last report"); io.f64(rep.device_ms, "last report");
        io.vec(g.last_candidates_, "last candidates");
        io.f64(center[0], "window centre"); io.f64(center[1], "window centre");
        io.check(!finite_se2(g.correction_) || !finite_se2(g.prev_) || !std::isfinite(g.accdist_) || !std::isfinite(g.factordist_) || !finite(center, 2),
                 "non-finite graph state");
        // key poses: every one at least 136 bytes before its points
        io.length(g.keys_, 4 + 2 * 32 + 7 * 8 + 8 + 4, "key poses");
        for (size_t i = 0; i < g.keys_.size() && io.ok(); ++i) {
            GraphSlam2D::KeyPose& k = g.keys_[i];
            io.i32(k.id, "key pose"); io.se2(k.pose, "key pose"); io.se2(k.original, "key pose");
            for (double& v : k.origin) io.f64(v, "key pose");
            for (double& v : k.quat) io.f64(v, "key pose");
            io.f64(k.stamp, "key pose");
            io.vec(k.pts, "key points", 3);
            io.check(k.id != (int)i, "a key pose id differs from its index");
            io.check(!finite_se2(k.pose) || !finite_se2(k.original) || !finite(k.origin, 3) || !finite(k.quat, 4), "non-finite key pose");
        }
        const size_t n = g.keys_.size();
        auto is_key = [n](int v) { return v >= 0 && (size_t)v < n; };
        io.length(g.links_, 8, "links");
        for (auto& l : g.links_) { io.i32(l.first, "links"); io.i32(l.second, "links"); }
        // the pose graph
        io.length(g.priors_, 4 + 4 * 8 + 4 * 8, "priors");
        for (PgoPrior& p : g.priors_) {
            io.i32(p.node, "priors"); io.se2(p.measured, "priors");
            loss(io, p.loss, "priors");
            io.check(!is_key(p.node), "a prior names no key");
            io.check(!finite_se2(p.measured), "non-finite prior");
        }
        betweens(io, g.factors_, n, "factors");
        betweens(io, g.queue_, n, "loop-factor queue");
        for (const auto& l : g.links_) io.check(!is_key(l.first) || !is_key(l.second), "a link names no key");
        for (int v : g.last_candidates_) io.check(!is_key(v), "a loop candidate names no key");
        io.check(g.mapping_keyid_ > n, "mapping key id past the key poses");
    }
};

// ---- the entry points --------------------------------------------------------------------------------------------------------------
int PFSlam2D::save(const std::string& path, CheckpointStats* st)
{
    SaveFrame f(st);
    if (opt_.shard_count > 1) return fail("saveState: a sharded handle cannot be saved (each rank holds only its part of the filter)", LAMA_ERR_STATE);
    return Ckpt::save_pf(*this, path, false, f);
}

int PFSlam2D::save_shard(const std::string& path, CheckpointStats* st)
{
    SaveFrame f(st);
    if (opt_.shard_count < 2) return fail("saveShardState: the handle is not sharded; save it with lama_pf_save_state", LAMA_ERR_STATE);
    if (pending_maps_)
        return fail("saveShardState: the handle is inside a split-phase step (between shard_begin and shard_map_update); save after shard_map_update",
                    LAMA_ERR_STATE);
    return Ckpt::save_pf(*this, path, true, f);
}

PFSlam2D* PFSlam2D::load(const std::string& path, const DeviceOptions& dev, std::string& err, int* code, CheckpointStats* st)
{
    return load_sharded({path}, 0, 1, dev, err, code, st, true);
}

PFSlam2D* PFSlam2D::load_sharded(const std::vector<std::string>& paths, uint32_t shard_rank, uint32_t shard_count, const DeviceOptions& dev,
                                 std::string& err, int* code, CheckpointStats* st, bool whole_only)
{
    LoadFrame f(st, code, err);
    if (paths.empty()) { err = "no checkpoint files"; return nullptr; }
    if (shard_count < 1 || shard_rank >= shard_count) { err = "shard_rank must be below shard_count (>= 1)"; return nullptr; }
    std::vector<Ckpt::ShardSource> src;
    const Ckpt::ShardSource* first = nullptr;   // the shared sections come from the first file
    const Ckpt::ShardSource* own = nullptr;     // the rank-local fields from this rank's file at the saved world size
    uint32_t per = 0, lo = 0;
    for (size_t i = 0; i < paths.size(); ++i) {
        Ckpt::ShardSource so;
        if (!Ckpt::read_source(f, paths[i], whole_only, paths.size() > 1, so, err)) return nullptr;
        if (i == 0) {
            PFOptions o = so.h->opt_;
            o.shard_rank = shard_rank; o.shard_count = shard_count;
            if (!PFSlam2D::valid_options(o, err)) return nullptr;
            per = o.particles / shard_count;
            lo = shard_rank * per;
            src.resize(so.count);
        } else if (!Ckpt::same_set(so, *first, err)) {
            return nullptr;
        }
        Ckpt::ShardSource& at = src[so.rank];
        if (at.h) { err = "shard rank " + std::to_string(so.rank) + " appears twice"; return nullptr; }
        at = std::move(so);
        if (i == 0) first = &at;
        if (at.count == shard_count && at.rank == shard_rank) own = &at;
        Ckpt::take_particles(at, lo, per);
        f.parsed();
    }
    for (size_t k = 0; k < src.size(); ++k)
        if (!src[k].h) { err = "shard rank " + std::to_string(k) + " is missing from the set"; return nullptr; }
    // the device options: dir_dim and max_beams 0 or the saved values; pool_slots too at the saved world size, any value at another
    const bool same_world = own != nullptr, present = first->has_engine;
    DeviceOptions check = dev;
    if (!same_world) check.pool_slots = 0;
    if (!geometry_matches(check, first->h->opt_.dev, present ? &first->img : nullptr, err)) return nullptr;
    const int capacity = shard_count > 1 ? 2 * (int)per : (int)per;
    EngineImage img;
    if (present) {
        img = first->img;
        img.particles = (int)per;
        if (same_world) {
            std::copy(own->img.counters, own->img.counters + 3, img.counters);
        } else {
            img.pool_slots = dev.pool_slots > 0 ? dev.pool_slots : Engine::auto_pool_slots(capacity);
            std::fill(img.counters, img.counters + 3, 0);
        }
        if (!Ckpt::assemble(src, img, err)) return nullptr;
    }
    const PFSlam2D zero;
    Ckpt::copy_rank_local(*first->h, same_world ? *own->h : zero);
    std::unique_ptr<PFSlam2D> p = std::move(src[first->rank].h);
    p->opt_.shard_rank = shard_rank; p->opt_.shard_count = shard_count;
    p->opt_.dev.device = dev.device; p->opt_.dev.stream = dev.stream; p->opt_.dev.timing = dev.timing;
    if (!present && !same_world && dev.pool_slots > 0) p->opt_.dev.pool_slots = dev.pool_slots;
    p->place();
    if (!f.device()) return nullptr;
    if (present) {
        p->eng_.reset(f.restore(img, dev, capacity));
        if (!p->eng_) return nullptr;
    }
    return f.done(p);
}

int Slam2D::save(const std::string& path, CheckpointStats* st)
{
    SaveFrame f(st);
    const int rc = f.snapshot(eng_.get(), err_);
    if (rc != LAMA_OK) return rc;
    Ckpt::slam_sections(f.w, *this, opt_.lidar_odometry);
    return f.write(path, opt_.lidar_odometry ? kCkptLidarOdometry2D : kCkptSlam2D, err_);
}

Slam2D* Slam2D::load(const std::string& path, const DeviceOptions& dev, std::string& err, int* code, CheckpointStats* st)
{
    LoadFrame f(st, code, err);
    std::vector<uint8_t> file;
    uint32_t kind = 0;
    if (!f.read(path, file, &kind)) return nullptr;
    if (kind != kCkptSlam2D && kind != kCkptLidarOdometry2D) { err = wrong_kind(kind, "Slam2D"); return nullptr; }
    std::unique_ptr<Slam2D> p(new Slam2D());
    CkptReader r = ckpt_body(file);
    Ckpt::slam_sections(r, *p, kind == kCkptLidarOdometry2D);
    EngineImage img;
    bool present = false;
    if (r.ok()) ckpt_get_engine(r, &present, img, 1, p->opt_.occupancy == 1 ? 1 : 0);
    r.check(p->has_first_ && !present, "a Slam2D past its first scan without device state");
    if (!f.checked(r) || !geometry_matches(dev, p->opt_.dev, present ? &img : nullptr, err)) return nullptr;
    f.parsed();
    if (!Ckpt::restore_slam(f, *p, present ? &img : nullptr, dev, err)) return nullptr;
    return f.done(p);
}

int GraphSlam2D::save(const std::string& path, CheckpointStats* st)
{
    SaveFrame f(st);
    int rc = f.snapshot(slam_->engine(), err_);
    // the global map only when the next generate_occupancy_map would draw on it
    if (rc == LAMA_OK) rc = f.snapshot(mapping_keyid_ > 0 && occ_ ? occ_->engine() : nullptr, err_);
    if (rc != LAMA_OK) return rc;
    double c[2];
    slam_->window_center(c);
    Ckpt::graph_sections(f.w, *this, c);
    return f.write(path, kCkptGraphSlam2D, err_);
}

GraphSlam2D* GraphSlam2D::load(const std::string& path, const DeviceOptions& dev, std::string& err, int* code, CheckpointStats* st)
{
    LoadFrame f(st, code, err);
    std::vector<uint8_t> file;
    uint32_t kind = 0;
    if (!f.read(path, file, &kind)) return nullptr;
    if (kind != kCkptGraphSlam2D) { err = wrong_kind(kind, "GraphSlam2D"); return nullptr; }
    std::unique_ptr<GraphSlam2D> p(new GraphSlam2D());
    p->slam_.reset(new Slam2D());
    Slam2D& s = *p->slam_;
    CkptReader r = ckpt_body(file);
    double center[2];
    Ckpt::graph_sections(r, *p, center);
    EngineImage inner, gimg;
    bool inner_present = false, global_present = false;
    if (r.ok()) ckpt_get_engine(r, &inner_present, inner, 1, 0, false);
    r.check(inner_present && inner.known_plane, "the inner engine has a known plane");
    r.check((s.has_first_ || !p->keys_.empty()) && !inner_present, "a GraphSlam2D past its first scan without device state");
    if (r.ok()) ckpt_get_engine(r, &global_present, gimg, 1, 0, true);
    r.check(global_present && !gimg.known_plane, "the global map's engine has no known plane");
    r.check(global_present != (p->mapping_keyid_ > 0), "a global map section must be present exactly when the mapping key id is above 0");
    if (!f.checked(r) || !geometry_matches(dev, s.opt_.dev, inner_present ? &inner : nullptr, err)) return nullptr;
    f.parsed();
    if (!Ckpt::restore_slam(f, s, inner_present ? &inner : nullptr, dev, err)) return nullptr;
    if (s.eng_) s.eng_->set_center(center[0], center[1]);
    p->opt_.slam = s.opt_;   // with the device pgo_optimize_graph runs on
    if (global_present) {
        Engine* e = f.restore(gimg, dev);
        if (!e) return nullptr;
        p->occ_.reset(OccupancyMapDev::adopt(e, s.opt_.dev.pool_slots <= 0));
        p->occ_->set_follow(true);
    }
    return f.done(p);
}

}  // namespace lama_b200
