// dev_common.cuh -- parameter blocks, counters and sm_90a PTX helpers shared by the kernels of libb200bpe.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "bpe_tables.h"
#include "text_access.cuh"

namespace b2bpe {

// device-side error / retry flags (Counters::err)
static const uint32_t ERR_NOBYTE = 1u;      // a piece needs a single-byte token the vocabulary lacks (lib.rs:202,207)
static const uint32_t ERR_DOCOFF = 2u;      // malformed document offsets
static const uint32_t ERR_BADTOKEN = 4u;    // decode: unknown token id
static const uint32_t ERR_LONGCAP = 8u;     // long-piece merge scratch too small for this batch  -> host grows it and re-runs
static const uint32_t ERR_MISSCAP = 16u;    // miss queue / miss result space too small            -> host grows it and re-runs
static const uint32_t ERR_SLOWCAP = 64u;    // list of positions for the general rule function too small               -> host grows it and re-runs
static const uint32_t ERR_INTERNAL = 128u;  // a kernel invariant did not hold (reported, never silently wrong)
static const uint32_t ERR_SPECIAL = 32u;    // a disallowed special token occurs in the text (tiktoken/core.py:120-124)

struct UcTables {
    const uint16_t *stage1; const uint8_t *stage2; const uint8_t *ascii;
    uint32_t one;            // == 1, opaque to the compiler: keeps v * one + c an IMAD (FMA pipe) in the pre-tokeniser's byte tests
};

static const int N_CLS = 8;                  // length classes of pieces longer than SHORT_MAX (see LongQ::cls)
static const int CLS_G1024 = 4, CLS_WARP = 5, CLS_BLOCK = 6, CLS_CLUSTER = 7;

struct Counters {            // device-resident, zeroed per call; copied to pinned host memory at the end of a pipeline
    unsigned long long long_bytes;   // bytes of pieces that merge in the global scratch (exact, even past the capacity)
    unsigned long long miss_bytes;   // sum of the lengths of the missed pieces = size of their result space (exact)
    unsigned long long total_tokens;
    unsigned long long special_pos;  // byte offset of the first disallowed special (ERR_SPECIAL)
    unsigned int n_long;
    unsigned int n_cls[10];          // long pieces per length class ([N_CLS]: pieces that did not fit the merge scratch)
    unsigned int cls_head[10];       // work-queue heads of the per-class kernels
    unsigned int n_big;
    unsigned int n_miss;             // exact, even past the capacity
    unsigned int n_cut;              // allowed-special occurrences found by the device scan
    unsigned int n_doc_tiles;        // sub-tiles that contain a document start (sparse-document batches)
    unsigned int n_slow;             // positions left to the general rule function (exact, even past the capacity)
    unsigned int special_idx;        // which disallowed special (ERR_SPECIAL)
    unsigned int ticket;
    unsigned int err;
    unsigned int n_owner;            // missed pieces that are merged: one per distinct piece, plus the unplaced and 16-byte ones
    unsigned int n_unplaced;         // missed pieces of <= 15 bytes the miss memo did not place (no key, no empty slot, or memo full)
};

static const uint32_t GROUP_MAX = 1024;       // pieces up to this length merge in shared memory, a group of lanes per piece
static const uint32_t BLOCK_MIN = 4096;       // pieces longer than this get a whole block
static const uint32_t CLUSTER_MIN = 32768;    // pieces longer than this get a thread-block cluster (8 x 1024 threads)
static const uint32_t LONG_SCRATCH_MIN = 256; // pieces longer than this merge in global scratch (warp / block / cluster per piece)

struct LongQ {               // queue of pieces longer than SHORT_MAX bytes
    unsigned long long *start;   // byte offset of the piece
    unsigned int *len;
    unsigned long long *off;     // offset of its region in the global merge scratch (pieces > LONG_SCRATCH_MIN only)
    unsigned int *ntok;
    // indices (into this queue) per length class: 0: 17..32, 1: 33..64, 2: 65..128, 3: 129..256, 4: 257..GROUP_MAX bytes
    // (a group of lanes per piece), 5: ..BLOCK_MIN (warp per piece, global scratch), 6: ..CLUSTER_MIN (block per piece),
    // 7: longer (cluster per piece)
    unsigned int *cls[N_CLS];
    unsigned long long scratch_cap;   // capacity (entries) of the global merge scratch
    uint32_t *sub_count;              // tokens per 1 KiB sub-tile: a finished piece credits its tokens to the sub-tile of its start
};

// a long piece is done: publish its token count (the gather reads ntok, the scan reads sub_count)
__device__ __forceinline__ void long_piece_done(const LongQ &q, unsigned int qi, uint32_t nt) {
    q.ntok[qi] = nt;
    atomicAdd(q.sub_count + (q.start[qi] >> 10), nt);
}

struct LongScratch {
    uint32_t *idA, *rkA, *idB, *rkB, *aux1, *aux2;
    uint8_t *flag;
};

struct SmemCol32 {           // per-lane column of a [k][32] shared-memory array: bank == lane whatever k is
    uint32_t *base;
    __device__ __forceinline__ uint32_t &operator[](int j) const { return base[j * 32]; }
};

__device__ __forceinline__ uint32_t warp_min_u32(uint32_t v) {
    return __reduce_min_sync(0xFFFFFFFFu, v);
}
__device__ __forceinline__ uint32_t warp_sum_u32(uint32_t v) {
    return __reduce_add_sync(0xFFFFFFFFu, v);
}
__device__ __forceinline__ uint32_t warp_incl_scan_u32(uint32_t v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, v, o); if (lane >= o) v += y; }
    return v;
}

// ---- cache-policy loads / stores -------------------------------------------------------------------------
// Streaming data (text, bit masks, slot arrays, results) must not push the rank tables out of L1: they are read
// with L1::no_allocate and written with evict-first (st.global.cs) hints; the tables stay on the default path.
__device__ __forceinline__ uint4 ld_stream_u4(const void *p) {
    uint4 v;
    asm("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint32_t ld_stream_u32(const void *p) {
    uint32_t v;
    asm("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ U4 ld_stream_U4(const U4 *p) {
    const uint4 v = ld_stream_u4(p);
    U4 r; r.x = v.x; r.y = v.y; r.z = v.z; r.w = v.w; return r;
}
__device__ __forceinline__ void st_stream_u32(uint32_t *p, uint32_t v) { __stcs(p, v); }
__device__ __forceinline__ void st_stream_u4(uint4 *p, uint4 v) { __stcs(p, v); }

// ---- 128-bit single-copy-atomic load and compare-and-swap (sm_90: LDG.E.128.STRONG.GPU, ATOMG.E.CAS.128) ----------
__device__ __forceinline__ uint4 u4_of(unsigned long long lo, unsigned long long hi) {
    return make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
}
__device__ __forceinline__ uint4 ld_relaxed_b128(const uint4 *p) {
    unsigned long long lo, hi;
    asm volatile("{\n\t.reg .b128 t;\n\tld.relaxed.gpu.global.b128 t, [%2];\n\tmov.b128 {%0, %1}, t;\n\t}"
                 : "=l"(lo), "=l"(hi) : "l"(p) : "memory");
    return u4_of(lo, hi);
}
// stores v at p if *p == 0; returns the old value (0: stored)
__device__ __forceinline__ uint4 cas_zero_b128(uint4 *p, uint4 v) {
    unsigned long long lo, hi;
    const unsigned long long vlo = (unsigned long long)v.y << 32 | v.x, vhi = (unsigned long long)v.w << 32 | v.z, z = 0;
    asm volatile("{\n\t.reg .b128 c, v, r;\n\tmov.b128 c, {%2, %2};\n\tmov.b128 v, {%3, %4};\n\t"
                 "atom.relaxed.gpu.global.cas.b128 r, [%5], c, v;\n\tmov.b128 {%0, %1}, r;\n\t}"
                 : "=l"(lo), "=l"(hi) : "l"(z), "l"(vlo), "l"(vhi), "l"(p) : "memory");
    return u4_of(lo, hi);
}

// ---- mbarrier + TMA 1-D bulk copy (cp.async.bulk, SASS UBLKCP) -------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t mbar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t mbar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(mbar), "r"(parity) : "memory");
    } while (!done);
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
// global -> shared bulk copy by the TMA unit; dst, src 16-byte aligned, bytes a multiple of 16; completes on mbar
__device__ __forceinline__ void tma_load_1d(uint32_t dst_smem, const void *src, uint32_t bytes, uint32_t mbar, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(mbar), "l"(pol) : "memory");
}

// low-`bits` mask, bits clamped to [0, 32] by the shifter (SHF.L.W with clamp)
__device__ __forceinline__ uint32_t low_mask_clamped(int bits) {
    return __funnelshift_lc(0xFFFFFFFFu, 0u, (uint32_t)max(bits, 0));
}

}  // namespace b2bpe
