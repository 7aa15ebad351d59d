// ddm3_check.cpp -- a standalone comparison of the host build of ddm3_core.h (ddm3_emu.cpp) with the oracle (ddm3_oracle.cpp) on
// one scenario file, built with -fsanitize=address,undefined by tests/ddm3_oracle.py so that the core's scenarios also run under
// the sanitizers.  Exit status 0 when every comparison holds.
//   usage: ddm3_check <scenario> <resolution> <l2_max> <wx> <wy> <wz> <pool_slots>
// The scenario is little-endian uint32 words: steps of {0, n, n ops of x y z kind} (a batch) or {1} (an update).  After every
// update both maps must agree on processed, the patch set, the bounds and every cell of every patch.
// TEST INFRASTRUCTURE ONLY.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <set>
#include <vector>

extern "C" {
void* d3o_create(double resolution, double l2_max);
void d3o_destroy(void* h);
void d3o_apply(void* h, const uint32_t* ops, int n);
uint32_t d3o_update(void* h);
int d3o_bounds(void* h, uint32_t* mn, uint32_t* mx);
int d3o_patch_ids(void* h, uint64_t* ids);
void d3o_export(void* h, const uint32_t* lo, const int32_t* size, uint64_t* words, uint8_t* known);
void* d3e_create(double resolution, double l2_max, const double* center, const int32_t* window, int pool_slots);
void d3e_destroy(void* h);
int d3e_apply(void* h, const uint32_t* ops, int n);
int d3e_update(void* h, uint32_t* processed);
int d3e_bounds(void* h, uint32_t* mn, uint32_t* mx);
int d3e_patch_ids(void* h, uint64_t* ids);
void d3e_export(void* h, const uint32_t* lo, const int32_t* size, uint64_t* words, uint8_t* known);
}

int main(int argc, char** argv)
{
    if (argc != 8) { std::fprintf(stderr, "usage: ddm3_check <scenario> <resolution> <l2_max> <wx> <wy> <wz> <pool_slots>\n"); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    std::vector<uint32_t> s;
    uint32_t w;
    while (std::fread(&w, 4, 1, f) == 1) s.push_back(w);
    std::fclose(f);
    const double res = std::atof(argv[2]), l2 = std::atof(argv[3]);
    const int32_t win[3] = {std::atoi(argv[4]), std::atoi(argv[5]), std::atoi(argv[6])};
    void* o = d3o_create(res, l2);
    void* e = d3e_create(res, l2, nullptr, win, std::atoi(argv[7]));
    const uint64_t uc = 2642244ull, uc2 = uc * uc;
    int updates = 0, bad = 0;
    for (size_t i = 0; i < s.size() && !bad;) {
        if (s[i] == 0) {
            const int n = (int)s[i + 1];
            const uint32_t* ops = s.data() + i + 2;
            if (d3e_apply(e, ops, n) != 0) { std::fprintf(stderr, "batch refused\n"); bad = 1; break; }
            d3o_apply(o, ops, n);
            i += 2 + 4 * (size_t)n;
            continue;
        }
        ++i;
        ++updates;
        uint32_t pe = 0;
        const int rc = d3e_update(e, &pe);
        const uint32_t po = d3o_update(o);
        if (rc != 0 || pe != po) { std::fprintf(stderr, "update %d: rc %d processed %u vs %u\n", updates, rc, pe, po); bad = 1; break; }
        uint32_t mno[3], mxo[3], mne[3], mxe[3];
        const int no = d3o_bounds(o, mno, mxo), ne = d3e_bounds(e, mne, mxe);
        std::vector<uint64_t> io((size_t)no), ie((size_t)ne);
        d3o_patch_ids(o, io.data());
        d3e_patch_ids(e, ie.data());
        if (std::set<uint64_t>(io.begin(), io.end()) != std::set<uint64_t>(ie.begin(), ie.end())) { std::fprintf(stderr, "update %d: patch sets differ\n", updates); bad = 1; break; }
        for (int k = 0; k < 3 && no; ++k)
            if (mno[k] != mne[k] || mxo[k] != mxe[k]) { std::fprintf(stderr, "update %d: bounds differ\n", updates); bad = 1; }
        std::vector<uint64_t> wo(32768), we(32768);
        std::vector<uint8_t> ko(32768), ke(32768);
        const int32_t size[3] = {32, 32, 32};
        for (uint64_t id : io) {
            const uint32_t lo[3] = {(uint32_t)((id / uc2) << 5), (uint32_t)(((id % uc2) / uc) << 5), (uint32_t)((id % uc) << 5)};
            d3o_export(o, lo, size, wo.data(), ko.data());
            d3e_export(e, lo, size, we.data(), ke.data());
            if (wo != we || ko != ke) { std::fprintf(stderr, "update %d: cells of patch %llu differ\n", updates, (unsigned long long)id); bad = 1; break; }
        }
    }
    d3o_destroy(o);
    d3e_destroy(e);
    if (!bad) std::printf("ok: %d updates\n", updates);
    return bad;
}
