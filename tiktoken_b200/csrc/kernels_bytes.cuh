// kernels_bytes.cuh -- bytes mode (b200bpe_encode_bytes_batch): documents that need not be UTF-8, with the semantics
// of CoreBPE::_encode_bytes (src/py.rs:72-115) and _increase_last_piece_token_len (src/lib.rs:444-481).
//
// Per document b with v = valid_up_to(b) < len(b), the reference encodes b[..v] as its own haystack, drops the tokens
// of its last regex piece (extended backwards over all-space tokens when the first of them is all-space) and encodes
// the dropped bytes plus b[v..] as ONE piece.  On the device, inside the normal pipeline (run 1):
//
//   utf8_check_kernel    first ill-formed byte of every document -> vup[d] (atomicMin)
//   bytes_cut_kernel     a damaged document gets a haystack start at v, interior bits over (v, end) and one
//                        placeholder slot at v -- the machinery of an accepted special token, so run 1 pre-tokenises
//                        the prefix as its own haystack and never merges the tail
//   bytes_repair_kernel  after the gather: walks back over the document's tokens to the start u of the unstable
//                        piece, the number k of tokens to drop (placeholder included) and the tail length end - u
//
// then the host runs the pipeline again over the tails in "every document is one piece" mode (run 2), after
//
//   bytes_gather_kernel  tails [u_d, end_d) -> one compact buffer (run 2's text)
//
// and splices: bytes_count_kernel + the scan + bytes_splice_kernel (run-1 tokens minus the last k, then run-2 tokens).
#pragma once
#include "dev_common.cuh"
#include "utf8_check.cuh"

using namespace b2bpe;

static const uint32_t VUP_NONE = 0xFFFFFFFFu;      // vup[d]: the document is well-formed

struct BytesCounters {       // bytes_repair_kernel, per run 1; zeroed with vup, copied to pinned host memory with Counters
    unsigned int n_docs;             // documents that are not well-formed UTF-8
    unsigned int pad;
    unsigned long long drop;         // run-1 tokens they drop (placeholders included)
    unsigned long long tail;         // bytes of their unstable pieces (run 2's text)
};

// document that contains byte pos (the last d with doc_off[d] <= pos; empty documents never contain a byte)
__device__ __forceinline__ unsigned long long doc_of(const unsigned long long *__restrict__ doc_off, unsigned long long n_docs,
                                                     const uint32_t *__restrict__ dbits, const uint32_t *__restrict__ span_first_doc,
                                                     unsigned long long pos) {
    const long long w = (long long)(pos >> 5);
    unsigned long long lo = 0, hi = n_docs;         // doc_off[lo] <= pos < doc_off[hi]
    if (dbits[w] & ((2u << (pos & 31)) - 1u)) lo = span_first_doc[w];   // a document starts in this span at or before pos
    else {
        while (hi - lo > 1) {
            const unsigned long long mid = (lo + hi) >> 1;
            if (doc_off[mid] <= pos) lo = mid; else hi = mid;
        }
        return lo;
    }
    while (doc_off[lo + 1] <= pos) lo++;
    return lo;
}

__global__ void __launch_bounds__(256) utf8_check_kernel(const uint8_t *__restrict__ text, long long n_bytes,
                                                        const uint32_t *__restrict__ dbits, const uint32_t *__restrict__ span_first_doc,
                                                        const unsigned long long *__restrict__ doc_off, unsigned long long n_docs,
                                                        long long n_words, uint32_t *vup) {
    const long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (w >= n_words) return;
    uint32_t m = utf8_bad_word(text, n_bytes, dbits, w);
    while (m) {                                     // the first mark of each document that has one in this span
        const unsigned long long pos = (unsigned long long)w * 32 + (unsigned)(__ffs(m) - 1);
        const unsigned long long d = doc_of(doc_off, n_docs, dbits, span_first_doc, pos);
        atomicMin(&vup[d], (uint32_t)pos);
        const unsigned long long end = doc_off[d + 1];
        if (end >= (unsigned long long)w * 32 + 32) break;
        m &= ~((1u << (uint32_t)(end - (unsigned long long)w * 32)) - 1u);
    }
}

// one warp per document: the cut at v (haystack start, placeholder slot, no piece start inside the tail)
__global__ void __launch_bounds__(256) bytes_cut_kernel(const unsigned long long *__restrict__ doc_off, unsigned long long n_docs,
                                                       const uint32_t *__restrict__ vup, uint32_t *hbits, uint32_t *ibits,
                                                       uint32_t *sbits, uint32_t *ltok) {
    const unsigned long long d = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    const uint32_t v = vup[d];
    if (v == VUP_NONE) return;
    const unsigned long long end = doc_off[d + 1];
    if (lane == 0) {
        atomicOr(&hbits[v >> 5], 1u << (v & 31));
        atomicOr(&sbits[v >> 5], 1u << (v & 31));
        ltok[v] = 0;                                // placeholder id: dropped by the splice
    }
    const unsigned long long a = (unsigned long long)v + 1;      // interior (v, end)
    if (a >= end) return;
    for (unsigned long long wi = (a >> 5) + lane; wi <= ((end - 1) >> 5); wi += 32) {
        const unsigned long long lo = max(a, wi * 32), hi = min(end, wi * 32 + 32);
        const uint32_t bits = (uint32_t)((hi - lo == 32 ? 0xFFFFFFFFull : ((1ull << (hi - lo)) - 1ull)) << (lo - wi * 32));
        if (bits == 0xFFFFFFFFu) ibits[wi] = bits;  // a whole word of this tail: no other document touches it
        else atomicOr(&ibits[wi], bits);
    }
}

// token id -> byte length through the decode tables (as decode_len_kernel reads them)
__device__ __forceinline__ uint32_t tok_len(const uint32_t *__restrict__ tok_boff, uint32_t n_ids, uint32_t t) {
    return t < n_ids ? __ldg(tok_boff + t + 1) - __ldg(tok_boff + t) : 0u;
}
__device__ __forceinline__ bool tok_all_space(const uint32_t *__restrict__ space_bits, uint32_t n_ids, uint32_t t) {
    return t < n_ids && ((__ldg(space_bits + (t >> 5)) >> (t & 31)) & 1u);
}

// The highest piece start in [start, v), 32 pbits words per warp step; start when there is none.  Every lane returns it.
__device__ __forceinline__ unsigned long long last_piece_start(int lane, unsigned long long start, unsigned long long v,
                                                               const uint32_t *__restrict__ pbits) {
    long long p = -1;
    for (long long wb = (long long)((v - 1) >> 5); wb >= (long long)(start >> 5) && p < 0; wb -= 32) {
        const long long wi = wb - lane;
        uint32_t m = 0;
        if (wi >= (long long)(start >> 5)) {
            m = pbits[wi];
            const long long lo = (long long)start - wi * 32, hi = (long long)v - wi * 32;   // keep bits [lo, hi)
            if (hi < 32) m &= (1u << hi) - 1u;
            if (lo > 0) m &= ~((1u << lo) - 1u);
        }
        const uint32_t hit = __ballot_sync(0xFFFFFFFFu, m != 0);
        if (hit) {
            const int src = __ffs(hit) - 1;                  // the lane with the highest word
            const uint32_t mw = __shfl_sync(0xFFFFFFFFu, m, src);
            p = (wb - src) * 32 + (31 - __clz(mw));
        }
    }
    return p < 0 ? start : (unsigned long long)p;
}

// The tokens [t0, t1) of a haystack end at byte v and its last piece starts at p: L = the tokens from t1 - 1 backwards
// that cover [p, v), extended backwards over all-space tokens when the first of them is all-space
// (_increase_last_piece_token_len, lib.rs:455-476); bytes = what the L tokens cover.  False when p is not a token
// boundary (a kernel invariant).  One warp; every lane returns the same.
__device__ __forceinline__ bool last_piece_tokens(int lane, unsigned long long p, unsigned long long v,
                                                  const uint32_t *__restrict__ tokens, unsigned long long t0, unsigned long long t1,
                                                  const uint32_t *__restrict__ tok_boff, const uint32_t *__restrict__ space_bits,
                                                  uint32_t n_ids, unsigned long long &L_out, unsigned long long &bytes_out) {
    const unsigned long long plen = v - p;
    unsigned long long acc = 0, L = 0;
    bool ok = true;
    for (unsigned long long it = 0;; it += 32) {
        const long long ti = (long long)t1 - 1 - (long long)it - lane;
        const bool have = ti >= (long long)t0;
        const uint32_t len = have ? tok_len(tok_boff, n_ids, tokens[ti]) : 0u;
        const uint32_t inc = warp_incl_scan_u32(len, lane);
        const uint32_t reach = __ballot_sync(0xFFFFFFFFu, have && acc + inc >= plen);
        if (reach) {
            const int j = __ffs(reach) - 1;
            ok = acc + __shfl_sync(0xFFFFFFFFu, inc, j) == plen;   // a piece start is a token boundary
            L = it + j + 1;
            break;
        }
        if (!__all_sync(0xFFFFFFFFu, have)) { ok = false; break; }
        acc += __shfl_sync(0xFFFFFFFFu, inc, 31);
    }
    unsigned long long bytes = plen;
    if (ok && tok_all_space(space_bits, n_ids, tokens[t1 - L])) {   // _increase_last_piece_token_len
        for (;;) {
            const long long ti = (long long)(t1 - L) - 1 - lane;
            const bool sp = ti >= (long long)t0 && tok_all_space(space_bits, n_ids, tokens[ti]);
            const uint32_t len = sp ? tok_len(tok_boff, n_ids, tokens[ti]) : 0u;
            const uint32_t run = ~__ballot_sync(0xFFFFFFFFu, sp);
            const int n_sp = run ? __ffs(run) - 1 : 32;      // leading all-space tokens of this step
            bytes += __reduce_add_sync(0xFFFFFFFFu, lane < n_sp ? len : 0u);
            L += (unsigned long long)n_sp;
            if (n_sp < 32) break;
        }
    }
    L_out = L; bytes_out = bytes;
    return ok;
}

// One warp per document, after run 1's gather.  For a damaged document: p = the last piece start in [start, v),
// L = the tokens that cover [p, v), extended backwards over all-space tokens when the first of them is all-space
// (lib.rs:455-476); k = L + 1 tokens to drop (the placeholder is the last), u = v - (bytes of the L tokens).
// Writes kdrop[d] and tail[d] = end - u for every document (0 and 0 when it is well-formed).
__global__ void __launch_bounds__(256) bytes_repair_kernel(const unsigned long long *__restrict__ doc_off, unsigned long long n_docs,
                                                          uint32_t *vup, const uint32_t *__restrict__ pbits,
                                                          const uint32_t *__restrict__ tokens, const unsigned long long *__restrict__ tok_off,
                                                          const uint32_t *__restrict__ tok_boff, const uint32_t *__restrict__ space_bits,
                                                          uint32_t n_ids, uint32_t *kdrop, uint32_t *tail, BytesCounters *bc,
                                                          Counters *ctr) {
    const unsigned long long d = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    const uint32_t v = vup[d];
    if (v == VUP_NONE) { if (lane == 0) { kdrop[d] = 0; tail[d] = 0; } return; }
    const unsigned long long start = doc_off[d], end = doc_off[d + 1];
    const unsigned long long t1 = tok_off[d + 1] - 1;            // the placeholder; the prefix's tokens are [t0, t1)
    const unsigned long long t0 = tok_off[d];
    unsigned long long u = v, k = 1;
    bool ok = true;
    if (v > start) {
        const unsigned long long p = last_piece_start(lane, start, v, pbits);
        unsigned long long L = 0, bytes = 0;
        ok = last_piece_tokens(lane, p, v, tokens, t0, t1, tok_boff, space_bits, n_ids, L, bytes);
        u = v - bytes;
        k = L + 1;
    }
    if (lane == 0) {
        if (!ok) atomicOr(&ctr->err, ERR_INTERNAL);
        kdrop[d] = (uint32_t)k;
        tail[d] = (uint32_t)(end - u);
        atomicAdd(&bc->n_docs, 1u);
        atomicAdd(&bc->drop, k);
        atomicAdd(&bc->tail, (unsigned long long)(end - u));
        vup[d] = (uint32_t)u;                         // from here on: the unstable piece's start, for bytes_gather_kernel
    }
}

// run 2's text: the tails [u_d, end_d) back to back (toff = exclusive scan of tail[]); 16 output bytes per thread
__global__ void __launch_bounds__(256) bytes_gather_kernel(const uint8_t *__restrict__ text, unsigned long long n_docs,
                                                          const uint32_t *__restrict__ ustart,
                                                          const unsigned long long *__restrict__ toff, uint8_t *__restrict__ out) {
    const unsigned long long total = toff[n_docs];
    const unsigned long long q0 = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) * 16;
    if (q0 >= total) return;
    unsigned long long lo = 0, hi = n_docs;           // toff[lo] <= q0 < toff[hi]
    while (hi - lo > 1) {
        const unsigned long long mid = (lo + hi) >> 1;
        if (toff[mid] <= q0) lo = mid; else hi = mid;
    }
    unsigned long long d = lo;
    const unsigned long long q1 = min(total, q0 + 16);
    for (unsigned long long q = q0; q < q1; q++) {
        while (toff[d + 1] <= q) d++;
        out[q] = text[(unsigned long long)ustart[d] + (q - toff[d])];
    }
}

// final token count per document
__global__ void __launch_bounds__(256) bytes_count_kernel(const unsigned long long *__restrict__ off1, const unsigned long long *__restrict__ off2,
                                                         const uint32_t *__restrict__ kdrop, unsigned long long n_docs, uint32_t *cnt) {
    const unsigned long long d = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (d < n_docs) cnt[d] = (uint32_t)((off1[d + 1] - off1[d]) - kdrop[d] + (off2[d + 1] - off2[d]));
}

// one block per document: run-1 tokens minus the last kdrop, then the run-2 tokens, at base[d]
__global__ void __launch_bounds__(256) bytes_splice_kernel(const uint32_t *__restrict__ tok1, const unsigned long long *__restrict__ off1,
                                                          const uint32_t *__restrict__ tok2, const unsigned long long *__restrict__ off2,
                                                          const uint32_t *__restrict__ kdrop, const unsigned long long *__restrict__ base,
                                                          unsigned long long n_docs, uint32_t *__restrict__ out) {
    for (unsigned long long d = blockIdx.x; d < n_docs; d += gridDim.x) {
        const unsigned long long a = off1[d], n1 = off1[d + 1] - a - kdrop[d], b = off2[d], n2 = off2[d + 1] - b;
        uint32_t *dst = out + base[d];
        for (unsigned long long i = threadIdx.x; i < n1; i += blockDim.x) dst[i] = tok1[a + i];
        for (unsigned long long i = threadIdx.x; i < n2; i += blockDim.x) dst[n1 + i] = tok2[b + i];
    }
}
