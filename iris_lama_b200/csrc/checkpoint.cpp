// checkpoint.cpp -- framing, checksum and the engine section of PFSlam2D / Slam2D checkpoints (format: checkpoint.h, DESIGN.md §13).
#include "checkpoint.h"

#include <chrono>
#include <cstdio>
#include <sstream>

namespace lama_b200 {

namespace {
double ms_since(std::chrono::steady_clock::time_point a) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count(); }
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

void ckpt_put_engine(CkptWriter& w, const EngineImage* img)
{
    if (img && !img->parked.empty()) w.version = kCkptVersionParked;
    w.u8(img != nullptr);
    if (!img) return;
    w.i32(img->particles); w.i32(img->dir_dim); w.i32(img->pool_slots); w.i32(img->max_beams); w.i32(img->occupancy_kind);
    w.u8(img->known_plane);
    w.f64(img->resolution); w.f64(img->l2_max);
    w.i32(img->window.base_px); w.i32(img->window.base_py);
    for (int k = 0; k < 3; ++k) w.u64(img->counters[k]);
    w.u32(img->used);
    w.bytes(img->refcount.data(), img->refcount.size() * 4);
    w.bytes(img->dirs.data(), img->dirs.size() * 4);
    if (w.version == kCkptVersionParked) {
        const size_t n_lists = (size_t)img->particles * img->n_kinds();
        for (size_t li = 0; li < n_lists; ++li) w.u32(li < img->park_len.size() ? (uint32_t)img->park_len[li] : 0u);
        for (const ParkEntry& e : img->parked) { w.i32(e.px); w.i32(e.py); w.i32(e.entry); }
    }
}

bool ckpt_get_engine(CkptReader& r, bool* present, EngineImage& img, int particles, int occupancy_kind, bool last)
{
    *present = r.u8("engine flag");
    if (!r.ok() || !*present) return r.ok();
    img.particles = r.i32("particles"); img.dir_dim = r.i32("dir_dim"); img.pool_slots = r.i32("pool_slots"); img.max_beams = r.i32("max_beams");
    img.occupancy_kind = r.i32("occupancy kind");
    img.known_plane = r.u8("known plane");
    img.resolution = r.f64("resolution"); img.l2_max = r.f64("l2_max");
    img.window.dim = img.dir_dim;
    img.window.base_px = r.i32("window"); img.window.base_py = r.i32("window");
    for (int k = 0; k < 3; ++k) img.counters[k] = r.u64("store counters");
    img.used = r.u32("used slots");
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

}  // namespace lama_b200
