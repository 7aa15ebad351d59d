// checkpoint.h -- the file format of PFSlam2D / Slam2D / GraphSlam2D checkpoints (host only, no CUDA).
//
// Little endian.  A 32-byte header {u64 magic "LAMACKPT", u32 format version, u32 handle kind, u64 total file size, u64 FNV-1a-64 of every
// byte after the header}, then the sections: options (field by field), front-end state, and the engine section -- u8 present, then
// geometry, window, store counters, K, K reference counts, the directories of every particle and kind, and the K slot payloads.  A
// GraphSlam2D file holds two engine sections, each followed by its own slot payloads.
// Version 2 (written only when a map has parked entries, window_shift_core.h; everything else is still written as version 1): the body
// starts with the 8-byte marker "LAMAPARK", and every engine section carries, between its directories and its slots, the parked lists:
// particles x kinds u32 lengths, then the entries {i32 patch x, i32 patch y, i32 directory entry} list after list.
// The byte-exact layout is in DESIGN.md §13; tests/test_checkpoint.py, tests/test_graph_checkpoint.py and tests/test_shard_checkpoint.py
// write it independently.  checkpoint.cpp states every section once, as a template over CkptWriter / CkptReader that save and load
// share, and holds the save / load entry points of PFSlam2D, Slam2D and GraphSlam2D.
#pragma once

#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "engine.h"

namespace lama_b200 {

constexpr uint64_t kCkptMagic      = 0x54504B43414D414Cull;   // "LAMACKPT"
constexpr uint32_t kCkptVersion    = 1;
constexpr uint32_t kCkptVersionParked = 2;
constexpr uint64_t kCkptParkMarker = 0x4B524150414D414Cull;   // "LAMAPARK"
constexpr size_t kCkptHeaderBytes  = 32;
// kind 5 is one rank's shard of a sharded PFSlam2D: {u32 shard_rank, u32 shard_count, u64 session id}, then the options and state
// sections of kind 1, then the engine section of the rank's own particles (DESIGN.md §13)
enum CkptKind : uint32_t { kCkptPFSlam2D = 1, kCkptSlam2D = 2, kCkptLidarOdometry2D = 3, kCkptGraphSlam2D = 4, kCkptPFSlam2DShard = 5 };

// what the last save / load took (ms) and moved
struct CheckpointStats {
    CheckpointTimes dev;
    double encode_ms = 0, io_ms = 0, total_ms = 0;   // encode: serialisation + checksum (save) / checksum + parsing + checks (load); io: file write / read
    uint64_t used_slots = 0, references = 0, file_bytes = 0;
};

// The field vocabulary a section is written in once, as a template over CkptWriter and CkptReader: every method takes its field by
// reference, writes it (writer) or reads it into place (reader).  check(bad, message) is a reader's refusal and does nothing in a writer;
// kLoad tells the few places where the two directions differ apart.
class CkptWriter {
public:
    static constexpr bool kLoad = false;
    std::vector<uint8_t> buf = std::vector<uint8_t>(kCkptHeaderBytes, 0);
    uint32_t version = kCkptVersion;   // ckpt_put_engine raises it to kCkptVersionParked for an image with parked entries
    bool ok() const { return true; }
    size_t pos() const { return buf.size(); }
    void check(bool, const char*, const char* = nullptr) {}
    void bytes(const void* p, size_t n) { const uint8_t* b = (const uint8_t*)p; buf.insert(buf.end(), b, b + n); }
    template <typename T> void put(T v) { bytes(&v, sizeof(T)); }   // the hosts this builds for are little endian
    void u8(bool v, const char* = nullptr) { put<uint8_t>(v ? 1 : 0); }
    void u32(uint32_t v, const char* = nullptr) { put(v); }
    void i32(int32_t v, const char* = nullptr) { put(v); }
    void u64(uint64_t v, const char* = nullptr) { put(v); }
    void f64(double v, const char* = nullptr) { put(v); }
    void se2(const SE2& s, const char* = nullptr) { f64(s.c); f64(s.s); f64(s.tx); f64(s.ty); }
    void str(const std::string& s, const char* = nullptr) { u32((uint32_t)s.size()); bytes(s.data(), s.size()); }
    // n elements of v in one copy
    template <typename T> void array(const std::vector<T>& v, size_t n, const char*) { bytes(v.data(), n * sizeof(T)); }
    // u32 v.size() / group, then all of v in one copy
    template <typename T> void vec(const std::vector<T>& v, const char*, size_t group = 1) { u32((uint32_t)(v.size() / group)); array(v, v.size(), nullptr); }
    // u32 v.size(): the length of a list whose elements follow field by field
    template <typename T> void length(const std::vector<T>& v, size_t, const char*) { u32((uint32_t)v.size()); }
};

// Bounds-checked reads: a read past the end sets the error and reads zeros, so a parser can check once per section.
class CkptReader {
public:
    static constexpr bool kLoad = true;
    CkptReader(const uint8_t* p, size_t n, uint32_t version = kCkptVersion) : version(version), p_(p), n_(n) {}
    uint32_t version;
    bool ok() const { return err_.empty(); }
    const std::string& error() const { return err_; }
    void fail(const std::string& m) { if (err_.empty()) err_ = m; }
    // the first refusal wins; `what` is appended in parentheses
    void check(bool bad, const char* m, const char* what = nullptr)
    {
        if (ok() && bad) fail(what ? std::string(m) + " (" + what + ")" : std::string(m));
    }
    size_t left() const { return n_ - off_; }
    size_t pos() const { return off_; }
    const uint8_t* take(size_t n, const char* what)
    {
        if (!ok() || n > left()) { fail(std::string("truncated checkpoint (") + what + ")"); return nullptr; }
        const uint8_t* q = p_ + off_;
        off_ += n;
        return q;
    }
    template <typename T> void get(T& v, const char* what) { v = T{}; if (const uint8_t* q = take(sizeof(T), what)) std::memcpy(&v, q, sizeof(T)); }
    void u8(bool& v, const char* what)
    {
        uint8_t b;
        get(b, what);
        if (b > 1) fail(std::string("bad flag byte (") + what + ")");
        v = b == 1;
    }
    void u32(uint32_t& v, const char* what) { get(v, what); }
    void i32(int32_t& v, const char* what) { get(v, what); }
    void u64(uint64_t& v, const char* what) { get(v, what); }
    void f64(double& v, const char* what) { get(v, what); }
    void se2(SE2& s, const char* what) { f64(s.c, what); f64(s.s, what); f64(s.tx, what); f64(s.ty, what); }
    void str(std::string& s, const char* what)
    {
        uint32_t n;
        u32(n, what);
        const size_t m = count(n, 1, what);
        const uint8_t* q = take(m, what);
        s = q ? std::string((const char*)q, m) : std::string();
    }
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
    template <typename T> void vec(std::vector<T>& v, const char* what, size_t group = 1)
    {
        uint32_t n;
        u32(n, what);
        array(v, group * count(n, group * sizeof(T), what), what);
    }
    template <typename T> void length(std::vector<T>& v, size_t elem, const char* what)
    {
        uint32_t n;
        u32(n, what);
        v.assign(count(n, elem, what), T{});
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
// Reads `path` into `file` and checks the header: magic, version (and a version-2 body's marker), size, checksum.  *kind = the handle kind.
int ckpt_read_file(const std::string& path, std::vector<uint8_t>& file, uint32_t* kind, std::string& err, CheckpointStats* st);
// a reader of the body of a file ckpt_read_file accepted: after the header (and the marker), with the file's version
CkptReader ckpt_body(const std::vector<uint8_t>& file);

// The engine section.  put writes everything but the slot payloads (the caller passes them as the file's tail); get reads and checks the
// whole section -- geometry, window, counts against the file size, directory entries (slot < K, known flag bits only), in a version-2
// file the parked lists (each strictly sorted, every entry outside the saved window, slot < K, known flag bits only), every reference
// count against its directory and parked references -- and points img.slot_bytes into the reader's buffer.  An image with parked
// entries raises w.version; the sections of a file must all be written with its final version (a file's first engine section is the
// only one that can hold parked entries).  `particles` / `occupancy_kind` are what
// the front end expects (-1: any).  With `last`, the section must end the file; otherwise other sections may follow its slots.
void ckpt_put_engine(CkptWriter& w, const EngineImage* img);
bool ckpt_get_engine(CkptReader& r, bool* present, EngineImage& img, int particles, int occupancy_kind, bool last = true);

// the text std::mt19937's operator<< writes: 624 state words and an index <= 624
bool ckpt_check_rng(const std::string& text);

}  // namespace lama_b200
