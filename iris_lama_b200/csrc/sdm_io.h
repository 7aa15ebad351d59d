// sdm_io.h -- the reference's on-disk sparse-dense map format (".sdm") and the grey images of sdm::export_to_png,
// produced from / consumed into device maps through their exported cell planes.
//
// Reference: Map::write / Map::read  src/sdm/map.cpp:490-575, IOHeader include/lama/sdm/map.h:95-103 (MAGIC :72, IO_VERSION :75),
// patch payload Container::write/read src/sdm/container.cpp:143-176 (cells, then the 1-bit-per-cell mask),
// DynamicDistanceMap::writeParameters src/sdm/dynamic_distance_map.cpp:200-208 (max_sqdist_); the occupancy maps write no
// parameters (frequency_occupancy_map.h:81-88, probabilistic_occupancy_map.h:78-85, simple_occupancy_map.h:74-81);
// image content src/sdm/export.cpp:46-96, pixel addressing include/lama/image.h:79-80.
#pragma once

#include <cstdint>
#include <string>
#include <vector>

namespace lama_b200 {

constexpr uint32_t kSdmMagic   = 0x6d64732e;  // map.h:72
constexpr uint16_t kSdmVersion = 0x0103;      // map.h:75

struct SdmHeader {   // the reference's IOHeader with its natural padding made explicit
    uint32_t magic;
    uint16_t version;
    uint16_t pad0;
    uint32_t cell_size;
    uint32_t patch_length;
    uint64_t num_patches;
    float resolution;
    uint8_t is_3d;
    uint8_t pad1[3];
};
static_assert(sizeof(SdmHeader) == 32, "IOHeader layout");

// cell layouts of the reference maps
#pragma pack(push, 1)
struct SdmDistanceCell {  // DynamicDistanceMap::distance_t, dynamic_distance_map.h:48-53
    int16_t obstacle[3];
    uint16_t sqdist;
    uint8_t valid_obstacle;
    uint8_t is_queued;
};
struct SdmFrequencyCell {  // frequency_occupancy_map.h:43-46
    uint16_t occupied;
    uint16_t visited;
};
#pragma pack(pop)
static_assert(sizeof(SdmDistanceCell) == 10 && sizeof(SdmFrequencyCell) == 4, "cell layout");

// A map as the file holds it: patches in file order, `cells` = num_patches * volume * cell_size bytes, volume / 64 mask words per
// patch; volume = 1024 cells, or 32 768 when header.is_3d.
struct SdmFile {
    SdmHeader header{};
    std::vector<uint8_t> params;   // what writeParameters emitted
    std::vector<uint64_t> ids;     // (x >> 5) * 2642244 + (y >> 5), map.h:153-161
    std::vector<uint8_t> cells;
    std::vector<uint64_t> masks;
};

// A dense window of exported cell planes (row-major, w * h, origin (x0, y0) in absolute cells, all multiples of 32).
struct SdmWindow {
    uint32_t x0 = 0, y0 = 0;
    int w = 0, h = 0;
};

bool sdm_write(const std::string& path, const SdmFile& f, std::string& err);
// expect_3d: the file must hold a 3-D map (is_3d = 1, 32 x 32 x 32 patches); otherwise a 2-D one
bool sdm_read(const std::string& path, uint32_t expect_cell_size, size_t n_params, SdmFile& f, std::string& err, bool expect_3d = false);

// planes -> file: one patch per 32x32 block that holds a known cell (a reference patch always has one: Map::get marks
// the touched cell, map.cpp:400-411)
void sdm_from_distance(const SdmWindow& win, float resolution, uint32_t max_sqdist, const uint16_t* sqdist, const uint8_t* valid, const uint8_t* known,
                       const int16_t* ox, const int16_t* oy, const uint8_t* queued, SdmFile& out);
void sdm_from_frequency(const SdmWindow& win, float resolution, const uint16_t* occupied, const uint16_t* visited, const uint8_t* known, SdmFile& out);
void sdm_from_logodds(const SdmWindow& win, float resolution, const float* prob, const uint8_t* known, SdmFile& out);
// file -> the smallest patch-aligned window holding all its patches; false when the file has no patches
bool sdm_window_of(const SdmFile& f, SdmWindow& win);
void sdm_to_distance(const SdmFile& f, const SdmWindow& win, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox, int16_t* oy, uint8_t* queued);

// export.cpp:46-73 / :75-96: `out` is win.w * win.h bytes
void sdm_occupancy_image_frequency(const SdmWindow& win, const uint16_t* occupied, const uint16_t* visited, const uint8_t* known, uint8_t* out);
void sdm_occupancy_image_logodds(const SdmWindow& win, const float* prob, const uint8_t* known, double thresh, uint8_t* out);
void sdm_distance_image(const SdmWindow& win, const uint16_t* sqdist, const uint8_t* valid, const uint8_t* known, uint32_t max_sqdist, double resolution,
                        uint8_t* out);

}  // namespace lama_b200
