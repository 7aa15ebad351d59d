// checkpoint.h -- the file format of PFSlam2D / Slam2D / GraphSlam2D checkpoints (host only, no CUDA).
//
// Little endian.  A 32-byte header {u64 magic "LAMACKPT", u32 format version, u32 handle kind, u64 total file size, u64 FNV-1a-64 of every
// byte after the header}, then the sections: options (field by field), front-end state, and the engine section -- u8 present, then
// geometry, window, store counters, K, K reference counts, the directories of every particle and kind, and the K slot payloads.  A
// GraphSlam2D file holds two engine sections, each followed by its own slot payloads.
// The byte-exact layout is in DESIGN.md §13; tests/test_checkpoint.py and tests/test_graph_checkpoint.py write it independently.
#pragma once

#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "engine.h"

namespace lama_b200 {

constexpr uint64_t kCkptMagic      = 0x54504B43414D414Cull;   // "LAMACKPT"
constexpr uint32_t kCkptVersion    = 1;
constexpr size_t kCkptHeaderBytes  = 32;
enum CkptKind : uint32_t { kCkptPFSlam2D = 1, kCkptSlam2D = 2, kCkptLidarOdometry2D = 3, kCkptGraphSlam2D = 4 };

// what the last save / load took (ms) and moved
struct CheckpointStats {
    CheckpointTimes dev;
    double encode_ms = 0, io_ms = 0, total_ms = 0;   // encode: serialisation + checksum (save) / checksum + parsing + checks (load); io: file write / read
    uint64_t used_slots = 0, references = 0, file_bytes = 0;
};

class CkptWriter {
public:
    std::vector<uint8_t> buf = std::vector<uint8_t>(kCkptHeaderBytes, 0);
    void bytes(const void* p, size_t n) { const uint8_t* b = (const uint8_t*)p; buf.insert(buf.end(), b, b + n); }
    template <typename T> void put(T v) { bytes(&v, sizeof(T)); }   // the hosts this builds for are little endian
    void u8(bool v) { put<uint8_t>(v ? 1 : 0); }
    void u32(uint32_t v) { put(v); }
    void i32(int32_t v) { put(v); }
    void u64(uint64_t v) { put(v); }
    void f64(double v) { put(v); }
    void se2(const SE2& s) { f64(s.c); f64(s.s); f64(s.tx); f64(s.ty); }
    void str(const std::string& s) { u32((uint32_t)s.size()); bytes(s.data(), s.size()); }
};

// Bounds-checked reads: a read past the end sets the error and returns zeros, so a parser can check once per section.
class CkptReader {
public:
    CkptReader(const uint8_t* p, size_t n) : p_(p), n_(n) {}
    bool ok() const { return err_.empty(); }
    const std::string& error() const { return err_; }
    void fail(const std::string& m) { if (err_.empty()) err_ = m; }
    size_t left() const { return n_ - off_; }
    const uint8_t* take(size_t n, const char* what)
    {
        if (!ok() || n > left()) { fail(std::string("truncated checkpoint (") + what + ")"); return nullptr; }
        const uint8_t* q = p_ + off_;
        off_ += n;
        return q;
    }
    template <typename T> T get(const char* what) { T v{}; if (const uint8_t* q = take(sizeof(T), what)) std::memcpy(&v, q, sizeof(T)); return v; }
    bool u8(const char* what) { const uint8_t v = get<uint8_t>(what); if (v > 1) fail(std::string("bad flag byte (") + what + ")"); return v == 1; }
    uint32_t u32(const char* what) { return get<uint32_t>(what); }
    int32_t i32(const char* what) { return get<int32_t>(what); }
    uint64_t u64(const char* what) { return get<uint64_t>(what); }
    double f64(const char* what) { return get<double>(what); }
    SE2 se2(const char* what) { SE2 s; s.c = f64(what); s.s = f64(what); s.tx = f64(what); s.ty = f64(what); return s; }
    // an element count whose elements (elem bytes each) must still fit in the file: checked before anything is allocated
    size_t count(uint64_t n, size_t elem, const char* what)
    {
        if (ok() && (elem ? n > left() / elem : n > left())) fail(std::string("count exceeds the file (") + what + ")");
        return ok() ? (size_t)n : 0;
    }
    template <typename T> void array(std::vector<T>& v, size_t n, const char* what)
    {
        n = count(n, sizeof(T), what);
        v.assign(n, T{});
        if (const uint8_t* q = take(n * sizeof(T), what)) std::memcpy(v.data(), q, n * sizeof(T));
    }
    std::string str(const char* what)
    {
        const size_t n = count(u32(what), 1, what);
        const uint8_t* q = take(n, what);
        return q ? std::string((const char*)q, n) : std::string();
    }

private:
    const uint8_t* p_;
    size_t n_, off_ = 0;
    std::string err_;
};

uint64_t fnv1a64(const uint8_t* p, size_t n, uint64_t h = 1469598103934665603ull);

// bytes written after the serialisation buffer without being copied into it (slot payloads, and the sections between them)
struct CkptSegment {
    const uint8_t* p;
    size_t n;
};
// Fills the header of w.buf and writes w.buf, then the `tail` segments in order, to `path`; the checksum covers them all.
int ckpt_write_file(const std::string& path, uint32_t kind, CkptWriter& w, const std::vector<CkptSegment>& tail, std::string& err, CheckpointStats* st);
// Reads `path` into `file` and checks the header: magic, version, size, checksum.  *kind = the handle kind.
int ckpt_read_file(const std::string& path, std::vector<uint8_t>& file, uint32_t* kind, std::string& err, CheckpointStats* st);

// The engine section.  put writes everything but the slot payloads (the caller passes them as the file's tail); get reads and checks the
// whole section -- geometry, window, counts against the file size, directory entries (slot < K, known flag bits only), every reference
// count against its directory references -- and points img.slot_bytes into the reader's buffer.  `particles` / `occupancy_kind` are what
// the front end expects (-1: any).  With `last`, the section must end the file; otherwise other sections may follow its slots.
void ckpt_put_engine(CkptWriter& w, const EngineImage* img);
bool ckpt_get_engine(CkptReader& r, bool* present, EngineImage& img, int particles, int occupancy_kind, bool last = true);

// the text std::mt19937's operator<< writes: 624 state words and an index <= 624
bool ckpt_check_rng(const std::string& text);

}  // namespace lama_b200
