// om3d_core.h -- the per-cell updates and queries of the 3-D occupancy maps, shared by the sm_90a kernels (om3d.cu) and the host
// emulation tests.  Plain C++ usable from host and device.
//
// Reference: FrequencyOccupancyMap src/sdm/frequency_occupancy_map.cpp:38-172 (setFree :65-74, setOccupied :81-91, setUnknown
// :98-108, prune :149-158), ProbabilisticOccupancyMap src/sdm/probabilistic_occupancy_map.cpp:38-175 (setFree :82-91, setOccupied
// :98-107, setUnknown :114-123), the 3-D addressing of include/lama/sdm/map.h:125-189.
//
// A cell is one 32-bit word: {uint16 occupied; uint16 visited} (occupied in the low half) for a frequency map, the float bits of
// the log-odds for a probabilistic map.  The two uint16 counters wrap independently, as the reference's do.
#pragma once

#include "patch_window.h"
#include "ray_core.h"

namespace lama_b200 {

constexpr int kOm3Cells = kPatchCells * kPatchLen;   // 32 x 32 x 32 cells of 4 bytes per patch
constexpr int kOm3Log2Cells = 3 * kPatchLog2;
constexpr int kOm3KnownWords = kOm3Cells / 32;       // the Container mask: one bit per cell
constexpr int kOm3MaxEntries = 1 << 16;              // window entries: a record key (entry << 15 | cell) fits 31 bits

enum : int { kOm3Frequency = 0, kOm3LogOdds = 1 };
enum : uint32_t { kOm3SetFree = 0, kOm3SetOccupied = 1, kOm3SetUnknown = 2 };

// ---- frequency cells ------------------------------------------------------------------------------------------------------------
LAMA_HD uint32_t om3_freq_pack(uint32_t occupied, uint32_t visited) { return (occupied & 0xFFFFu) | ((visited & 0xFFFFu) << 16); }

// one setter of FrequencyOccupancyMap on the word; returns what the setter returns
LAMA_HD bool om3_freq_op(uint32_t& word, uint32_t op)
{
    uint32_t occ = occ_occupied(word), vis = occ_visited(word);
    if (op == kOm3SetUnknown) {        // :98-108
        if (vis == 0) return false;
        word = 0;
        return true;
    }
    if (op == kOm3SetOccupied) {       // :81-91
        const bool was = occ_is_occupied(occ, vis);
        occ = (occ + 1) & 0xFFFFu;
        vis = (vis + 1) & 0xFFFFu;
        word = om3_freq_pack(occ, vis);
        return !was && occ_is_occupied(occ, vis);
    }
    const bool was = occ_is_free(occ, vis);   // setFree :65-74
    vis = (vis + 1) & 0xFFFFu;
    word = om3_freq_pack(occ, vis);
    return !was && occ_is_free(occ, vis);
}

// ---- log-odds cells -------------------------------------------------------------------------------------------------------------
LAMA_HD float om3_bits_float(uint32_t w)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(w);
#else
    float f;
    __builtin_memcpy(&f, &w, 4);
    return f;
#endif
}
LAMA_HD uint32_t om3_float_bits(float f)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t w;
    __builtin_memcpy(&w, &f, 4);
    return w;
#endif
}

// one setter of ProbabilisticOccupancyMap on the float cell; returns what the setter returns
LAMA_HD bool om3_prob_op(float& p, uint32_t op, const ProbParams& pp)
{
    if (op == kOm3SetUnknown) {        // :114-123
        const bool unknown = (double)p == pp.thresh;
        p = (float)pp.thresh;
        return !unknown;
    }
    if (op == kOm3SetOccupied) {       // :98-107
        const bool was = (double)p > pp.thresh;
        p = prob_hit(p, pp);
        return !was && (double)p > pp.thresh;
    }
    const bool was = (double)p < pp.thresh;   // setFree :82-91
    p = prob_miss(p, pp);
    return !was && (double)p < pp.thresh;
}

// one op on a cell word of either kind
LAMA_HD bool om3_op(int kind, uint32_t& word, uint32_t op, const ProbParams& pp)
{
    if (kind == kOm3Frequency) return om3_freq_op(word, op);
    float p = om3_bits_float(word);
    const bool r = om3_prob_op(p, op, pp);
    word = om3_float_bits(p);
    return r;
}

// isFree / isOccupied / isUnknown as flag bits 0 / 1 / 2 of a cell that the const get() returns (`known`) or not (:110-147, :125-162)
LAMA_HD uint32_t om3_flags(int kind, bool known, uint32_t word, const ProbParams& pp)
{
    if (!known) return 4u;
    if (kind == kOm3Frequency) {
        const uint32_t occ = occ_occupied(word), vis = occ_visited(word);
        return (occ_is_free(occ, vis) ? 1u : 0u) | (occ_is_occupied(occ, vis) ? 2u : 0u) | (vis == 0 ? 4u : 0u);
    }
    const double p = (double)om3_bits_float(word);
    return (p < pp.thresh ? 1u : 0u) | (p > pp.thresh ? 2u : 0u) | (p == pp.thresh ? 4u : 0u);
}

// FrequencyOccupancyMap::prune's rule (:149-158) on one known cell
LAMA_HD uint32_t om3_prune(uint32_t word)
{
    const uint32_t occ = occ_occupied(word), vis = occ_visited(word);
    return (vis == 1 && occ <= 1) ? 0u : word;
}

// ---- the insertion of one point (generateOccupancyMap's body, graph_slam2d.cpp:146-158) ----------------------------------------
// setOccupied(w2m(hit)) first (step 0), then, with `full`, setFree on computeRay(so, w2m(hit)) (steps 1..), both ends excluded.
// from = so = w2m(tf.translation()), to = w2m(tf * p).
LAMA_HD BeamCells om3_point_cells(const Affine& tf, const double* pt, double scale)
{
    double hit[3];
    apply_tf(tf, pt[0], pt[1], pt[2], hit);
    BeamCells b;
    for (int k = 0; k < 3; ++k) {
        b.from[k] = w2m(tf.t[k], scale);
        b.to[k] = w2m(hit[k], scale);
    }
    b.mark_hit = true;
    return b;
}
// the records of one point: 1 + the interior cells of its ray
LAMA_HD uint32_t om3_point_records(const BeamCells& b, bool full)
{
    if (!full) return 1;
    const int a0 = (int)(b.to[0] - b.from[0]), a1 = (int)(b.to[1] - b.from[1]), a2 = (int)(b.to[2] - b.from[2]);
    int n = a0 < 0 ? -a0 : a0;
    n = (a1 < 0 ? -a1 : a1) > n ? (a1 < 0 ? -a1 : a1) : n;
    n = (a2 < 0 ? -a2 : a2) > n ? (a2 < 0 ? -a2 : a2) : n;
    return 1u + (n > 1 ? (uint32_t)(n - 1) : 0u);
}

}  // namespace lama_b200
