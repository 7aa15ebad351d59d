// sdm_io.cpp -- see sdm_io.h
#include "sdm_io.h"

#include <cmath>
#include <cstdio>
#include <cstring>

#include "lama_core.h"

namespace lama_b200 {

namespace {
constexpr uint64_t kUniversalConstant = 2642244ull;  // map.h:68
constexpr int kMaskWords = kPatchCells / 64;

struct File {
    FILE* f;
    explicit File(FILE* p) : f(p) {}
    ~File() { if (f) std::fclose(f); }
};

// every 32x32 block of the window with a known cell, in row-major block order
template <typename Emit>
void for_each_patch(const SdmWindow& win, const uint8_t* known, Emit&& emit)
{
    for (int by = 0; by < win.h / kPatchLen; ++by)
        for (int bx = 0; bx < win.w / kPatchLen; ++bx) {
            uint64_t mask[kMaskWords] = {0};
            bool any = false;
            for (int cy = 0; cy < kPatchLen; ++cy)
                for (int cx = 0; cx < kPatchLen; ++cx)
                    if (known[(size_t)(by * kPatchLen + cy) * win.w + bx * kPatchLen + cx]) {
                        const uint32_t ci = (uint32_t)cx | ((uint32_t)cy << kPatchLog2);  // map.h:182-189
                        mask[ci >> 6] |= 1ull << (ci & 63);                                // container.h:102-106
                        any = true;
                    }
            if (!any) continue;
            const uint64_t id = (uint64_t)((win.x0 >> kPatchLog2) + (uint32_t)bx) * kUniversalConstant + (uint64_t)((win.y0 >> kPatchLog2) + (uint32_t)by);
            emit(id, bx, by, mask);
        }
}
// cells of one patch: 32 x 32, or 32 x 32 x 32 when the header says is_3d (Map::read, map.cpp:550)
size_t patch_volume(const SdmHeader& h) { return (size_t)kPatchCells * (h.is_3d ? kPatchLen : 1); }
void begin_file(SdmFile& out, uint32_t cell_size, float resolution)
{
    out = SdmFile();
    out.header.magic        = kSdmMagic;
    out.header.version      = kSdmVersion;
    out.header.cell_size    = cell_size;
    out.header.patch_length = kPatchLen;
    out.header.resolution   = resolution;
    out.header.is_3d        = 0;
}
}  // namespace

bool sdm_write(const std::string& path, const SdmFile& f, std::string& err)
{
    File fp(std::fopen(path.c_str(), "wb"));
    if (!fp.f) { err = "cannot open " + path + " for writing"; return false; }
    const size_t vol = patch_volume(f.header), patch_bytes = vol * f.header.cell_size, mask_words = vol / 64;
    bool ok = std::fwrite(&f.header, sizeof(SdmHeader), 1, fp.f) == 1;
    if (ok && !f.params.empty()) ok = std::fwrite(f.params.data(), f.params.size(), 1, fp.f) == 1;
    for (size_t i = 0; ok && i < f.ids.size(); ++i) {
        ok = std::fwrite(&f.ids[i], 8, 1, fp.f) == 1 && std::fwrite(f.cells.data() + i * patch_bytes, patch_bytes, 1, fp.f) == 1 &&
             std::fwrite(f.masks.data() + i * mask_words, 8 * mask_words, 1, fp.f) == 1;
    }
    if (!ok) err = "short write to " + path;
    return ok;
}

bool sdm_read(const std::string& path, uint32_t expect_cell_size, size_t n_params, SdmFile& f, std::string& err, bool expect_3d)
{
    File fp(std::fopen(path.c_str(), "rb"));
    if (!fp.f) { err = "cannot open " + path; return false; }
    f = SdmFile();
    if (std::fread(&f.header, sizeof(SdmHeader), 1, fp.f) != 1) { err = "truncated header in " + path; return false; }
    if (f.header.magic != kSdmMagic || f.header.version != kSdmVersion) { err = "not an sdm file of version 0x0103: " + path; return false; }  // map.cpp:539
    if (f.header.cell_size != expect_cell_size || (f.header.is_3d != 0) != expect_3d) { err = "cell size / dimensionality mismatch in " + path; return false; }       // map.cpp:545
    if (f.header.patch_length != (uint32_t)kPatchLen) { err = "only 32-cell patches are supported: " + path; return false; }
    f.params.resize(n_params);
    if (n_params && std::fread(f.params.data(), n_params, 1, fp.f) != 1) { err = "truncated parameters in " + path; return false; }
    const size_t vol = patch_volume(f.header), patch_bytes = vol * f.header.cell_size, mask_words = vol / 64, n = (size_t)f.header.num_patches;
    {   // num_patches comes from an untrusted file: it must fit what is left of it before anything is sized from it
        const long here = std::ftell(fp.f);
        if (here < 0 || std::fseek(fp.f, 0, SEEK_END) != 0) { err = "cannot size " + path; return false; }
        const long end = std::ftell(fp.f);
        if (end < here || std::fseek(fp.f, here, SEEK_SET) != 0) { err = "cannot size " + path; return false; }
        const size_t per_patch = 8 + patch_bytes + 8 * mask_words;
        if (f.header.num_patches > (uint64_t)(end - here) / per_patch) { err = "truncated patch list in " + path; return false; }  // map.cpp:567
    }
    f.ids.resize(n);
    f.cells.resize(n * patch_bytes);
    f.masks.resize(n * mask_words);
    for (size_t i = 0; i < n; ++i) {
        if (std::fread(&f.ids[i], 8, 1, fp.f) != 1 || std::fread(f.cells.data() + i * patch_bytes, patch_bytes, 1, fp.f) != 1 ||
            std::fread(f.masks.data() + i * mask_words, 8 * mask_words, 1, fp.f) != 1) {
            err = "truncated patch list in " + path;  // map.cpp:567
            return false;
        }
    }
    return true;
}

void sdm_from_distance(const SdmWindow& win, float resolution, uint32_t max_sqdist, const uint16_t* sqdist, const uint8_t* valid, const uint8_t* known,
                       const int16_t* ox, const int16_t* oy, const uint8_t* queued, SdmFile& out)
{
    begin_file(out, sizeof(SdmDistanceCell), resolution);
    out.params.resize(4);
    std::memcpy(out.params.data(), &max_sqdist, 4);  // dynamic_distance_map.cpp:200-203
    for_each_patch(win, known, [&](uint64_t id, int bx, int by, const uint64_t* mask) {
        out.ids.push_back(id);
        out.masks.insert(out.masks.end(), mask, mask + kMaskWords);
        const size_t base = out.cells.size();
        out.cells.resize(base + (size_t)kPatchCells * sizeof(SdmDistanceCell), 0);
        SdmDistanceCell* c = reinterpret_cast<SdmDistanceCell*>(out.cells.data() + base);
        for (int cy = 0; cy < kPatchLen; ++cy)
            for (int cx = 0; cx < kPatchLen; ++cx) {
                const size_t k = (size_t)(by * kPatchLen + cy) * win.w + bx * kPatchLen + cx;
                if (!known[k]) continue;   // never written: the calloc'd zeros of Container::alloc (container.cpp:78-95)
                SdmDistanceCell& d = c[cx | (cy << kPatchLog2)];
                d.obstacle[0] = ox[k]; d.obstacle[1] = oy[k]; d.obstacle[2] = 0;
                d.sqdist = sqdist[k]; d.valid_obstacle = valid[k] != 0; d.is_queued = queued[k] != 0;
            }
    });
    out.header.num_patches = out.ids.size();
}

void sdm_from_frequency(const SdmWindow& win, float resolution, const uint16_t* occupied, const uint16_t* visited, const uint8_t* known, SdmFile& out)
{
    begin_file(out, sizeof(SdmFrequencyCell), resolution);
    for_each_patch(win, known, [&](uint64_t id, int bx, int by, const uint64_t* mask) {
        out.ids.push_back(id);
        out.masks.insert(out.masks.end(), mask, mask + kMaskWords);
        const size_t base = out.cells.size();
        out.cells.resize(base + (size_t)kPatchCells * sizeof(SdmFrequencyCell), 0);
        SdmFrequencyCell* c = reinterpret_cast<SdmFrequencyCell*>(out.cells.data() + base);
        for (int cy = 0; cy < kPatchLen; ++cy)
            for (int cx = 0; cx < kPatchLen; ++cx) {
                const size_t k = (size_t)(by * kPatchLen + cy) * win.w + bx * kPatchLen + cx;
                c[cx | (cy << kPatchLog2)] = SdmFrequencyCell{occupied[k], visited[k]};
            }
    });
    out.header.num_patches = out.ids.size();
}

void sdm_from_logodds(const SdmWindow& win, float resolution, const float* prob, const uint8_t* known, SdmFile& out)
{
    begin_file(out, sizeof(float), resolution);
    for_each_patch(win, known, [&](uint64_t id, int bx, int by, const uint64_t* mask) {
        out.ids.push_back(id);
        out.masks.insert(out.masks.end(), mask, mask + kMaskWords);
        const size_t base = out.cells.size();
        out.cells.resize(base + (size_t)kPatchCells * sizeof(float), 0);
        float* c = reinterpret_cast<float*>(out.cells.data() + base);
        for (int cy = 0; cy < kPatchLen; ++cy)
            for (int cx = 0; cx < kPatchLen; ++cx) c[cx | (cy << kPatchLog2)] = prob[(size_t)(by * kPatchLen + cy) * win.w + bx * kPatchLen + cx];
    });
    out.header.num_patches = out.ids.size();
}

bool sdm_window_of(const SdmFile& f, SdmWindow& win)
{
    if (f.ids.empty()) return false;
    uint32_t lo[2] = {0xffffffffu, 0xffffffffu}, hi[2] = {0, 0};
    for (uint64_t id : f.ids) {  // Map::p2m, map.h:166-177
        const uint32_t px = (uint32_t)(id / kUniversalConstant), py = (uint32_t)(id % kUniversalConstant);
        lo[0] = px < lo[0] ? px : lo[0]; lo[1] = py < lo[1] ? py : lo[1];
        hi[0] = px > hi[0] ? px : hi[0]; hi[1] = py > hi[1] ? py : hi[1];
    }
    win.x0 = lo[0] << kPatchLog2; win.y0 = lo[1] << kPatchLog2;
    win.w  = (int)((hi[0] - lo[0] + 1) << kPatchLog2);
    win.h  = (int)((hi[1] - lo[1] + 1) << kPatchLog2);
    return true;
}

void sdm_to_distance(const SdmFile& f, const SdmWindow& win, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox, int16_t* oy, uint8_t* queued)
{
    const size_t n = (size_t)win.w * win.h;
    std::memset(sqdist, 0, n * 2); std::memset(valid, 0, n); std::memset(known, 0, n);
    std::memset(ox, 0, n * 2); std::memset(oy, 0, n * 2); std::memset(queued, 0, n);
    for (size_t i = 0; i < f.ids.size(); ++i) {
        const uint32_t px = (uint32_t)(f.ids[i] / kUniversalConstant), py = (uint32_t)(f.ids[i] % kUniversalConstant);
        const int bx = (int)(px - (win.x0 >> kPatchLog2)), by = (int)(py - (win.y0 >> kPatchLog2));
        const SdmDistanceCell* c = reinterpret_cast<const SdmDistanceCell*>(f.cells.data() + i * (size_t)kPatchCells * sizeof(SdmDistanceCell));
        const uint64_t* mask = f.masks.data() + i * kMaskWords;
        for (uint32_t ci = 0; ci < (uint32_t)kPatchCells; ++ci) {
            if (!((mask[ci >> 6] >> (ci & 63)) & 1ull)) continue;
            const size_t k = (size_t)(by * kPatchLen + (int)(ci >> kPatchLog2)) * win.w + bx * kPatchLen + (int)(ci & (kPatchLen - 1));
            known[k] = 1; sqdist[k] = c[ci].sqdist; valid[k] = c[ci].valid_obstacle; queued[k] = c[ci].is_queued;
            ox[k] = c[ci].obstacle[0]; oy[k] = c[ci].obstacle[1];
        }
    }
}

void sdm_occupancy_image_frequency(const SdmWindow& win, const uint16_t* occupied, const uint16_t* visited, const uint8_t* known, uint8_t* out)
{
    const size_t n = (size_t)win.w * win.h;
    for (size_t k = 0; k < n; ++k) {
        if (!known[k]) { out[k] = 90; continue; }                                                 // export.cpp:55
        const double p = visited[k] == 0 ? 0.25 : ((double)occupied[k]) / ((double)visited[k]);   // frequency_occupancy_map.cpp:40-45
        out[k] = p < 0.25 ? 255 : (p > 0.25 ? 0 : 127);                                           // export.cpp:64-69
    }
}
void sdm_occupancy_image_logodds(const SdmWindow& win, const float* prob, const uint8_t* known, double thresh, uint8_t* out)
{
    const size_t n = (size_t)win.w * win.h;
    for (size_t k = 0; k < n; ++k) {
        if (!known[k]) { out[k] = 90; continue; }
        out[k] = (double)prob[k] < thresh ? 255 : ((double)prob[k] > thresh ? 0 : 127);           // probabilistic_occupancy_map.cpp:130-149
    }
}
void sdm_distance_image(const SdmWindow& win, const uint16_t* sqdist, const uint8_t* valid, const uint8_t* known, uint32_t max_sqdist, double resolution,
                        uint8_t* out)
{
    const size_t n = (size_t)win.w * win.h;
    const double max_distance = std::sqrt((double)max_sqdist) * resolution;                        // dynamic_distance_map.cpp:155-158
    for (size_t k = 0; k < n; ++k) {
        if (!known[k]) { out[k] = 127; continue; }                                                // export.cpp:83
        const double d = std::sqrt((double)(valid[k] ? sqdist[k] : max_sqdist)) * resolution;    // dynamic_distance_map.cpp:140-147
        out[k] = (uint8_t)(d * 255 / max_distance);                                               // export.cpp:91
    }
}

}  // namespace lama_b200
