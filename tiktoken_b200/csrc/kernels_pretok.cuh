// kernels_pretok.cuh -- documents -> doc-start bitmask; UTF-8 bytes -> piece-start bitmask (the regex pre-tokeniser,
// src/lib.rs:363-366 `find_iter` over the pat_strs of tiktoken_ext/openai_public.py:12-14, :89, :104-114).
#pragma once
#include "dev_common.cuh"
#include "pretok_fast.cuh"

using namespace b2bpe;

// --------------------------------------------------------------------------------------------
// kernel 0: documents -> doc-start bitmask, first document index per 32-byte span
// --------------------------------------------------------------------------------------------
__global__ void mark_docs_kernel(const unsigned long long *__restrict__ doc_off, unsigned long long n_docs,
                                 unsigned long long n_bytes, uint32_t *dbits, uint32_t *span_first_doc,
                                 uint32_t *doc_tiles /* NULL: dense documents, no list */, Counters *ctr) {
    unsigned long long d = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (d > n_docs) return;                           // index n_docs is the end sentinel (== n_bytes)
    unsigned long long pos = doc_off[d];
    bool bad = pos > n_bytes || (d < n_docs && doc_off[d + 1] < pos) || (d == 0 && pos != 0) ||
               (d == n_docs && pos != n_bytes);
    if (bad) { atomicOr(&ctr->err, ERR_DOCOFF); return; }
    atomicOr(&dbits[pos >> 5], 1u << (pos & 31));
    atomicMin(&span_first_doc[pos >> 5], (uint32_t)d);
    // list of the 1 KiB sub-tiles that contain a document start (each once: by the first document that starts there)
    if (doc_tiles && (d == 0 || (doc_off[d - 1] >> 10) != (pos >> 10))) {
        const uint32_t peers = __activemask();
        const int lane = threadIdx.x & 31, leader = __ffs(peers) - 1;
        unsigned int base = 0;
        if (lane == leader) base = atomicAdd(&ctr->n_doc_tiles, (unsigned int)__popc(peers));
        base = __shfl_sync(peers, base, leader);
        doc_tiles[base + __popc(peers & ((1u << lane) - 1u))] = (uint32_t)(pos >> 10);
    }
}

// --------------------------------------------------------------------------------------------
// kernel 1: pre-tokeniser.  One thread per 32-byte span = one word of the piece-start bitmask.
// The positions the bit-parallel rules cannot decide locally go through the general rule function,
// which is long and branchy: when a lane holds more than one of them, the warp pools its undecided
// positions and deals them out one per lane, so that the function runs once per ~32 positions instead
// of once per (busiest lane's) position with most lanes idle.
// --------------------------------------------------------------------------------------------
static const int PRETOK_WARPS = 8;

// o200k's rule function is long (case / mark chains): one out-of-line copy serves both call sites; the
// two shorter ones are inlined.
__device__ __noinline__ bool slow_boundary_o200k(const TextAccess &t, long long pos) { return boundary_before<PAT_O200K>(t, pos); }

template <int PAT>
__device__ __forceinline__ bool slow_boundary(const TextAccess &t, long long pos) {
    if (PAT == PAT_O200K) return slow_boundary_o200k(t, pos);
    return boundary_before<PAT>(t, pos);
}

// Fast part: the bit-parallel rules decide all but a fraction of a percent of the positions (none on English text);
// the rest go to a global list.  Keeping the general rule function OUT of this kernel keeps its register
// count low and its warps convergent -- the function is long, branchy and walks along runs.
// CUT: bytes mode (a haystack may start right after an ill-formed lead byte, see classify_window)
template <int PAT, bool CUT = false>
__global__ void __launch_bounds__(PRETOK_WARPS * 32, PAT == PAT_O200K ? 4 : 5) pretok_kernel(const uint8_t *__restrict__ text, long long n_bytes,
                                                                  const uint32_t *__restrict__ dbits, UcTables uc,
                                                                  uint32_t *__restrict__ pbits, uint32_t *__restrict__ psum,
                                                                  long long n_words, const uint32_t *__restrict__ ibits,
                                                                  uint32_t *__restrict__ slow_list, uint32_t slow_cap, Counters *ctr) {
    __shared__ uint32_t s_cnt, s_base;
    const long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const TextAccess t{text, n_bytes, dbits, uc.stage1, uc.stage2, uc.ascii, uc.one};
    if (threadIdx.x == 0) s_cnt = 0;
    uint64_t b = 0, slow = 0;
    if (w < n_words) b = span_fast<PAT, CUT>(t, w, slow);
    uint32_t sm = (uint32_t)(slow >> 8);                // own positions only
    if (ibits && w < n_words) sm &= ~ibits[w];          // inside an accepted special token: no piece start, nothing to decide
    uint32_t word = 0;
    if (w < n_words) {
        word = span_word(t, w, b);
        if (ibits) word &= ~ibits[w];                   // no piece starts inside an accepted special token
        pbits[w] = word;
    }
    // summary bitmap: bit = "this word of pbits has a piece start" (lets find_long skip long runs 32x faster);
    // pretok_slow_kernel adds the bits of the words it touches
    const uint32_t nz = __ballot_sync(0xFFFFFFFFu, word != 0);
    if (lane == 0 && (w >> 5) <= ((n_words - 1) >> 5)) psum[w >> 5] = nz;
    // undecided positions -> global list: one shared-memory atomic per warp, one global atomic per block
    const uint32_t cnt = (uint32_t)__popc(sm);
    const uint32_t inc = warp_incl_scan_u32(cnt, lane);
    const uint32_t wtot = __shfl_sync(0xFFFFFFFFu, inc, 31);
    __syncthreads();
    uint32_t woff = 0;
    if (lane == 0 && wtot) woff = atomicAdd(&s_cnt, wtot);
    woff = __shfl_sync(0xFFFFFFFFu, woff, 0);
    __syncthreads();
    const uint32_t btot = s_cnt;
    if (btot == 0) return;                               // block-uniform
    if (threadIdx.x == 0) s_base = atomicAdd(&ctr->n_slow, btot);
    __syncthreads();
    if (cnt) {
        uint32_t o = s_base + woff + inc - cnt;
        if ((unsigned long long)s_base + btot > slow_cap) { atomicOr(&ctr->err, ERR_SLOWCAP); return; }   // the host re-runs with the exact size
        for (uint32_t mm = sm; mm; mm &= mm - 1) slow_list[o++] = (uint32_t)(w * 32 + (__ffs(mm) - 1));
    }
}

// Slow part: one listed position per thread through the general rule function boundary_before<PAT>().
template <int PAT>
__global__ void __launch_bounds__(256) pretok_slow_kernel(const uint8_t *__restrict__ text, long long n_bytes,
                                                         const uint32_t *__restrict__ dbits, UcTables uc,
                                                         uint32_t *pbits, uint32_t *psum, const uint32_t *__restrict__ slow_list,
                                                         uint32_t slow_cap, const Counters *ctr) {
    if (ctr->err & ERR_SLOWCAP) return;
    const uint32_t n = min(ctr->n_slow, slow_cap);
    const TextAccess t{text, n_bytes, dbits, uc.stage1, uc.stage2, uc.ascii};
    for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u) {
        const uint32_t pos = slow_list[i];
        if (slow_boundary<PAT>(t, (long long)pos)) {
            atomicOr(&pbits[pos >> 5], 1u << (pos & 31));
            atomicOr(&psum[pos >> 10], 1u << ((pos >> 5) & 31));
        }
    }
}

// single-piece mode: every document is one piece, P = D (encode_single_piece is its one-document case; the bytes mode's
// run 2 encodes the unstable piece of every damaged document this way)
__global__ void single_piece_bits_kernel(uint32_t *pbits, uint32_t *psum, const uint32_t *__restrict__ dbits, long long n_words) {
    long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    uint32_t word = 0;
    if (w < n_words) {
        word = dbits[w];
        pbits[w] = word;
    }
    const uint32_t nz = __ballot_sync(0xFFFFFFFFu, word != 0);
    if ((threadIdx.x & 31) == 0 && (w >> 5) <= ((n_words - 1) >> 5)) psum[w >> 5] = nz;
}
