// device_store.cuh -- device-resident sparse-dense map store: one patch pool shared by all particles
// and both map kinds, per-particle dense directories, reference-counted copy-on-write patches.
//
// Replaces, for the hot path, the reference's  std::unordered_map<uint64, COWPtr<Container>>
// (include/lama/sdm/map.h:109) + Container (include/lama/sdm/container.h:47-162) +
// COWPtr::detach (include/lama/cow_ptr.h:96-114).
#pragma once

#include <cuda_runtime.h>

#include "lama_core.h"

namespace lama_b200 {

struct StoreView {
    uint32_t* pool;       // n_slots * 1024 words
    uint32_t* fbits;      // n_slots * 32 words: obstacle-mirror bit of every cell (occupancy patches)
    uint32_t* kbits;      // n_slots * 32 words: Container 'known' bit of log-odds occupancy patches (null for frequency maps)
    int32_t* refcount;    // per slot
    int32_t* free_slots;  // stack of free slot ids
    int32_t* free_count;  // number of valid entries in free_slots
    int32_t* freed;       // slots released during this scan; merged into free_slots by k_merge_free
    int32_t* freed_count;
    uint32_t* status;     // sticky error bits (lama_core.h)
    uint64_t* counters;   // [0] patches allocated, [1] patches detached (COW copies), [2] patches freed
    int32_t* ray_ctrl;    // task counters of the pull ray cast (kernels.cuh RayPullView::ctrl), reset by k_merge_free
    int32_t n_slots;
    int32_t* dirs;        // [set][particle][kind][dim*dim]
    int32_t n_particles;
    int32_t n_kinds;      // 2 (occupancy, distance) or 3 (+ per-scan scratch counters of the log-odds map)
    DirWindow window;
};

enum MapKind : int { kMapOcc = 0, kMapDm = 1, kMapScratch = 2 };

// A directory entry is -1 (patch absent) or slot | flags:
//   kDirHot   persistent, occupancy directories only: the patch may hold cells whose obstacle-mirror bit is set
//             (the ray-cast kernel uses fire-and-forget RED atomics on all other patches)
//   kDirOwn   persistent: this particle is the ONLY owner of the slot (reference count verified to be 1), so the
//             patch can be written in place without looking at the count.  Set on allocation, on copy-on-write
//             detach and when a count of 1 is observed; cleared on every entry that k_copy_dirs shares.
// (kDirSlotMask, kDirHot and kDirOwn live in lama_core.h, where the host-side checkpoint reader checks entries too)

__device__ __forceinline__ int32_t* dir_of(const StoreView& s, int set, int particle, int kind)
{
    return s.dirs + (((size_t)set * s.n_particles + particle) * s.n_kinds + kind) * (size_t)(s.window.dim * s.window.dim);
}
__device__ __forceinline__ uint32_t* patch_ptr(const StoreView& s, int slot) { return s.pool + (size_t)slot * kPatchCells; }
__device__ __forceinline__ uint32_t* fbits_ptr(const StoreView& s, int slot) { return s.fbits + (size_t)slot * 32; }
__device__ __forceinline__ uint32_t* kbits_ptr(const StoreView& s, int slot) { return s.kbits + (size_t)slot * 32; }

// ---- slot allocation (one thread) -----------------------------------------------------------------------
__device__ __forceinline__ int alloc_slot(const StoreView& s)
{
    int i = atomicSub(s.free_count, 1) - 1;
    if (i < 0) {
        atomicAdd(s.free_count, 1);
        atomicOr(s.status, kErrPoolEmpty);
        return -1;
    }
    int slot = s.free_slots[i];
    s.refcount[slot] = 1;
    return slot;
}
// drop one reference; the slot goes to the deferred free list when it was the last one.
__device__ __forceinline__ void release_slot(const StoreView& s, int slot)
{
    int old = atomicSub(&s.refcount[slot], 1);
    if (old == 1) {
        int i = atomicAdd(s.freed_count, 1);
        s.freed[i] = slot;
        atomicAdd((unsigned long long*)&s.counters[2], 1ull);
    }
}

// ---- warp-cooperative patch fill / copy (16 B per lane per step) ---------------------------------------
__device__ __forceinline__ void warp_zero_patch(uint32_t* dst, int lane)
{
    uint4 z = make_uint4(0, 0, 0, 0);
    uint4* d = reinterpret_cast<uint4*>(dst);
#pragma unroll
    for (int i = 0; i < kPatchBytes / 16 / 32; ++i) d[i * 32 + lane] = z;
}
__device__ __forceinline__ void warp_copy_patch(uint32_t* dst, const uint32_t* src, int lane)
{
    const uint4* sp = reinterpret_cast<const uint4*>(src);
    uint4* d        = reinterpret_cast<uint4*>(dst);
#pragma unroll
    for (int i = 0; i < kPatchBytes / 16 / 32; ++i) d[i * 32 + lane] = __ldcg(sp + i * 32 + lane);
}

// Make directory entry `di` of a particle's map writable by this warp: allocate a zeroed patch on
// first touch (Map::get mutable, map.cpp:400-408) or detach a shared one (cow_ptr.h:104-114).
// Must be called by all 32 lanes of a warp with identical arguments; `dir_smem` is the staged copy
// of the directory, `dir_gmem` its home.  Returns the (now exclusive) slot or -1 when the pool is empty.
// (cold path: kept out of line so that the hot loops of the callers stay small)
static __device__ __noinline__ int warp_make_exclusive(const StoreView& s, int32_t* dir_smem, int32_t* dir_gmem, int di, int lane)
{
    const int entry = dir_smem[di];
    const int slot  = entry < 0 ? -1 : (entry & kDirSlotMask);
    const int keep  = entry < 0 ? 0 : (entry & kDirHot);
    if (slot < 0) {
        int ns = 0;
        if (lane == 0) {
            ns = alloc_slot(s);
            if (ns >= 0) atomicAdd((unsigned long long*)&s.counters[0], 1ull);
        }
        ns = __shfl_sync(0xffffffffu, ns, 0);
        if (ns < 0) return -1;
        warp_zero_patch(patch_ptr(s, ns), lane);
        fbits_ptr(s, ns)[lane] = 0u;
        if (s.kbits) kbits_ptr(s, ns)[lane] = 0u;
        __syncwarp();
        if (lane == 0) {
            dir_smem[di] = ns | keep | kDirOwn;
            dir_gmem[di] = ns | keep | kDirOwn;
        }
        __syncwarp();
        return ns;
    }
    if (entry & kDirOwn) return slot;
    int rc = 0;
    if (lane == 0) rc = atomicAdd(&s.refcount[slot], 0);
    rc = __shfl_sync(0xffffffffu, rc, 0);
    if (rc > 1) {
        int ns = 0;
        if (lane == 0) {
            ns = alloc_slot(s);
            if (ns >= 0) atomicAdd((unsigned long long*)&s.counters[1], 1ull);
        }
        ns = __shfl_sync(0xffffffffu, ns, 0);
        if (ns < 0) return -1;
        // The source stays immutable while we hold our reference: a sharer only writes in place once
        // it observes refcount == 1, which cannot happen before we drop ours below.
        warp_copy_patch(patch_ptr(s, ns), patch_ptr(s, slot), lane);
        fbits_ptr(s, ns)[lane] = __ldcg(fbits_ptr(s, slot) + lane);
        if (s.kbits) kbits_ptr(s, ns)[lane] = __ldcg(kbits_ptr(s, slot) + lane);
        __syncwarp();
        if (lane == 0) {
            dir_smem[di] = ns | keep | kDirOwn;
            dir_gmem[di] = ns | keep | kDirOwn;
            __threadfence();
            release_slot(s, slot);
        }
        __syncwarp();
        return ns;
    }
    if (lane == 0) {  // sole owner: remember it
        dir_smem[di] = entry | kDirOwn;
        dir_gmem[di] = entry | kDirOwn;
    }
    __syncwarp();
    return slot;
}

// ---- TMA bulk copy of a directory into shared memory (cp.async.bulk + mbarrier) ------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// bytes must be a multiple of 16, both addresses 16-byte aligned.
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// Stage `bytes` of global memory into shared memory with one TMA bulk copy issued by thread 0; all
// threads of the block return once the data has landed.  `bar` is a block-shared mbarrier.
__device__ __forceinline__ void block_stage_tma(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar, uint32_t parity)
{
    if (threadIdx.x == 0) {
        mbar_expect_tx(bar, bytes);
        // a single bulk copy moves at most 2^20-1... keep chunks <= 32 KiB for safety
        uint32_t off = 0;
        while (off < bytes) {
            uint32_t chunk = bytes - off > 32768u ? 32768u : bytes - off;
            tma_load_1d((char*)dst_smem + off, (const char*)src_gmem + off, chunk, bar);
            off += chunk;
        }
    }
    mbar_wait(bar, parity);
}

}  // namespace lama_b200
