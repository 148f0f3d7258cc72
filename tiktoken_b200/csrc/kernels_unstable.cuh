// kernels_unstable.cuh -- completion search (b200bpe_encode_with_unstable_batch): the semantics of
// CoreBPE::_encode_unstable_native (src/lib.rs:483-599) for every document of a batch.
//
// Run 1 is the normal pipeline with the special-token flags of the call; inside it
//
//   unstable_walk_kernel    a warp per document: the tokens L of the last regex piece of the final haystack (0 when the
//                           document is empty or ends with an allowed special), extended backwards over all-space
//                           mergeable tokens (lib.rs:444-481); U = the bytes they cover, the document's tail
//
// then, per chunk, on the chunk's device:
//
//   unstable_search_kernel  a warp per document, a lane per search item: (a) the tokens that start with U, (b) for every
//                           i with |U| - i <= the longest token, the tokens that start with U[i:] -- two binary searches
//                           in the token ids sorted by their bytes --, (c) the whitespace split of the last scalar
//   scans                   candidates per item -> candidate index (the enumeration order of lib.rs:537-596), candidate
//                           text bytes per item -> text offset
//   then in rounds of at most one chunk of candidate text:
//   unstable_round_kernel   the last candidate of the round (binary search on the monotone text offset)
//   unstable_meta_kernel    per candidate: its item, token, prefix length, whether U[:i] + bytes(t) is UTF-8
//                           (utf8_bad_word on the junction, a per-token flag for the rest); text lengths of the two runs
//   unstable_gather_kernel  the candidate text of each run, back to back
//   run 2                   UTF-8 candidates through the ordinary pipeline (encode_ordinary), the others and both parts of
//                           (c) through single-piece mode; a single-piece result that is one token whose own merges do
//                           not reach it is replaced by its byte_pair_encode (a per-engine table)
//   unstable_insert_kernel  per candidate: the tokens up to the first that reaches |U| bytes, their 64-bit hash with the
//                           document, insert into the open-addressing table, atomicMin of the candidate index
//   unstable_verify_kernel  the candidate whose index won its slot is a new completion; any other compares its tokens
//                           exactly with the winner (a true 64-bit collision is reported and the chunk re-runs with
//                           another seed)
//   unstable_write_kernel   the new completions, in candidate order, appended to the chunk's result
#pragma once
#include "dev_common.cuh"
#include "kernels_bytes.cuh"
#include "utf8_check.cuh"

using namespace b2bpe;

static const uint32_t UR_NONE = 0xFFFFFFFFu;        // ur_idx[id]: the token is reached by its own merges
static const uint32_t UERR_TABLE = 1u;              // the dedup table had no free slot within UNST_PROBES steps: grow, re-run
static const uint32_t UERR_COLLIDE = 2u;            // two different sequences share a 64-bit key: new seed, re-run
static const uint32_t UERR_BIG = 4u;                // candidate text of one item does not fit 32 bits
static const int UNST_PROBES = 64;

enum { UK_A = 0, UK_B = 1, UK_C = 2 };              // search item kinds: (a) whole U, (b) a suffix U[i:], (c) whitespace split
enum { UM_A = 0, UM_ORD = 1, UM_BPE = 2, UM_C = 3 }; // candidate modes: [t]; encode_ordinary(P); byte_pair_encode(P); (c)

struct UnstTables {             // per device, built by the first completion search of an engine
    const uint32_t *sorted;     // mergeable ids in byte order of their bytes (sorted_token_bytes, lib.rs:659-660)
    const unsigned long long *lenpre;   // prefix sums of their lengths (n_sorted + 1)
    uint32_t n_sorted;
    const uint32_t *tok_boff; const uint8_t *tok_blob; uint32_t n_ids;   // the decode tables
    const uint32_t *space;      // bit per id: a MERGEABLE token of ' ', '\n', '\t' only (self.decoder, lib.rs:455-465)
    const uint8_t *u8info;      // per id: bits 0-2 = leading continuation bytes (capped at 4), bit 3 = the rest is UTF-8
    const uint32_t *ur_idx;     // per id: UR_NONE, or the index of its byte_pair_encode in ur_off / ur_tok
    const uint32_t *ur_off; const uint32_t *ur_tok;
    uint32_t max_len;           // longest mergeable token
};

struct UnstCounters {           // per chunk, zeroed by the host
    unsigned long long n_docs;      // documents with unstable bytes
    unsigned long long n_encoded;   // candidates that went through run 2
    unsigned long long n_bpe;       // ... through byte_pair_encode (single-piece mode)
    unsigned long long round[2];    // unstable_round_kernel: last candidate, text bytes of the round
    unsigned long long tot[2];      // totals read back by the host (scan results)
    unsigned int err;               // UERR_*
    unsigned int pad;
};

__device__ __forceinline__ uint32_t ut_len(const UnstTables &U, uint32_t t) { return tok_len(U.tok_boff, U.n_ids, t); }
__device__ __forceinline__ const uint8_t *ut_bytes(const UnstTables &U, uint32_t t) { return U.tok_blob + __ldg(U.tok_boff + t); }

// Rust's char::is_whitespace (White_Space)
__device__ __forceinline__ bool unicode_white_space(uint32_t c) {
    return (c >= 0x09u && c <= 0x0Du) || c == 0x20u || c == 0x85u || c == 0xA0u || c == 0x1680u ||
           (c >= 0x2000u && c <= 0x200Au) || c == 0x2028u || c == 0x2029u || c == 0x202Fu || c == 0x205Fu || c == 0x3000u;
}

// One warp per document of run 1, after its gather: L (tokens of the last piece, extended), |U| and the number of search
// items (0 without unstable bytes; else (a), one (b) per i in [|U| - m, |U|) with m = min(|U| - 1, longest token), (c)).
__global__ void __launch_bounds__(256) unstable_walk_kernel(const unsigned long long *__restrict__ doc_off, unsigned long long n_docs,
                                                           const uint32_t *__restrict__ pbits, const uint32_t *__restrict__ sbits,
                                                           const uint32_t *__restrict__ tokens, const unsigned long long *__restrict__ tok_off,
                                                           const uint32_t *__restrict__ tok_boff, const uint32_t *__restrict__ space_bits,
                                                           uint32_t n_ids, uint32_t max_len, uint32_t *kdrop, uint32_t *ulen,
                                                           uint32_t *nitem, Counters *ctr) {
    const unsigned long long d = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    const unsigned long long start = doc_off[d], end = doc_off[d + 1];
    unsigned long long L = 0, bytes = 0;
    bool ok = true;
    if (end > start) {
        const unsigned long long p = last_piece_start(lane, start, end, pbits);
        // a document that ends with an allowed special has an empty final haystack: last_piece_token_len = 0 (lib.rs:433)
        if (!(sbits && ((sbits[p >> 5] >> (p & 31)) & 1u)))
            ok = last_piece_tokens(lane, p, end, tokens, tok_off[d], tok_off[d + 1], tok_boff, space_bits, n_ids, L, bytes);
    }
    if (lane == 0) {
        if (!ok) { atomicOr(&ctr->err, ERR_INTERNAL); L = 0; bytes = 0; }
        kdrop[d] = (uint32_t)L;
        ulen[d] = (uint32_t)bytes;
        nitem[d] = bytes ? (uint32_t)min(bytes - 1, (unsigned long long)max_len) + 2u : 0u;
    }
}

// -1 / 0 / +1: token t against the string s[0..n) in slice order; `prefix` makes every token that starts with s compare
// equal (the end of the range of lib.rs:541-543)
__device__ __forceinline__ int ut_cmp(const UnstTables &U, uint32_t t, const uint8_t *s, uint32_t n, bool prefix) {
    const uint8_t *b = ut_bytes(U, t);
    const uint32_t lt = ut_len(U, t), m = min(lt, n);
    for (uint32_t k = 0; k < m; k++) {
        const uint32_t x = b[k], y = s[k];
        if (x != y) return x < y ? -1 : 1;
    }
    if (lt < n) return -1;
    return (lt == n || prefix) ? 0 : 1;
}
// first sorted index whose token compares >= 0 (prefix = false) or > 0 (prefix = true) against s
__device__ __forceinline__ uint32_t ut_bound(const UnstTables &U, const uint8_t *s, uint32_t n, bool prefix) {
    uint32_t lo = 0, hi = U.n_sorted;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        const int c = ut_cmp(U, __ldg(U.sorted + mid), s, n, prefix);
        if (prefix ? c <= 0 : c < 0) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// start and length of the last scalar of U (U is well-formed: it is a suffix of a str from a piece start)
__device__ __forceinline__ uint32_t ut_last_scalar(const uint8_t *u, uint32_t n, uint32_t &cp) {
    uint32_t q = n - 1;
    while (q > 0 && (u[q] & 0xC0u) == 0x80u) q--;
    const uint32_t ls = n - q, b0 = u[q];
    cp = ls == 1 ? b0 : ls == 2 ? (b0 & 0x1Fu) : ls == 3 ? (b0 & 0x0Fu) : (b0 & 0x07u);
    for (uint32_t k = q + 1; k < n; k++) cp = cp << 6 | (u[k] & 0x3Fu);
    return ls;
}

// One warp per document, a lane per search item: the token range, candidate count and candidate text bytes of each.
__global__ void __launch_bounds__(256) unstable_search_kernel(UnstTables U, const uint8_t *__restrict__ text,
                                                             const unsigned long long *__restrict__ doc_off, unsigned long long n_docs,
                                                             const uint32_t *__restrict__ ulen, const unsigned long long *__restrict__ item_base,
                                                             uint32_t *it_lo, uint32_t *it_cnt, uint32_t *it_bytes, uint32_t *it_doc,
                                                             UnstCounters *uc) {
    const unsigned long long d = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (d >= n_docs) return;
    const uint32_t n = ulen[d];
    if (n == 0) return;
    if (lane == 0) atomicAdd(&uc->n_docs, 1ull);
    const uint8_t *u = text + doc_off[d + 1] - n;
    const unsigned long long k0 = item_base[d];
    const uint32_t nit = (uint32_t)(item_base[d + 1] - k0), m = nit - 2;
    for (uint32_t j = lane; j < nit; j += 32) {
        const unsigned long long k = k0 + j;
        uint32_t lo = 0, cnt = 0; unsigned long long bytes = 0;
        if (j + 1 < nit) {                               // (a): i = 0, (b): i = n - m + j - 1
            const uint32_t i = j == 0 ? 0u : n - m + j - 1;
            lo = ut_bound(U, u + i, n - i, false);
            cnt = ut_bound(U, u + i, n - i, true) - lo;
            if (j) bytes = (unsigned long long)cnt * i + (U.lenpre[lo + cnt] - U.lenpre[lo]);
        } else if (n > 1) {                              // (c), lib.rs:588-596
            uint32_t cp;
            const uint32_t ls = ut_last_scalar(u, n, cp);
            if (n > ls && unicode_white_space(cp)) { cnt = 1; bytes = n; }
        }
        if (bytes >= 0xFFFFFFFFull) { atomicOr(&uc->err, UERR_BIG); bytes = 0; }
        it_lo[k] = lo; it_cnt[k] = cnt; it_bytes[k] = (uint32_t)bytes; it_doc[k] = (uint32_t)d;
    }
}

struct UnstItems {              // search items of a chunk (k = item), their candidate and text bases (exclusive scans)
    const unsigned long long *doc_off; const uint32_t *ulen; const unsigned long long *item_base;
    const uint32_t *lo, *cnt, *doc;
    const unsigned long long *cbase, *tbase;   // n_items + 1
    unsigned long long n_items;
};

__device__ __forceinline__ unsigned long long ui_item_of(const UnstItems &I, unsigned long long c) {   // cbase[k] <= c < cbase[k + 1]
    unsigned long long lo = 0, hi = I.n_items;
    while (hi - lo > 1) {
        const unsigned long long mid = (lo + hi) >> 1;
        if (I.cbase[mid] <= c) lo = mid; else hi = mid;
    }
    return lo;
}
// kind of item k and its prefix length i
__device__ __forceinline__ int ui_kind(const UnstItems &I, unsigned long long k, uint32_t &i, uint32_t &n) {
    const uint32_t d = I.doc[k];
    n = I.ulen[d];
    const unsigned long long k0 = I.item_base[d];
    const uint32_t j = (uint32_t)(k - k0), nit = (uint32_t)(I.item_base[d + 1] - k0);
    if (j == 0) { i = 0; return UK_A; }
    if (j + 1 == nit) { i = n; return UK_C; }
    i = n - (nit - 2) + j - 1;
    return UK_B;
}
// text bytes of all candidates before candidate c (monotone in c)
__device__ __forceinline__ unsigned long long ui_text_before(const UnstTables &U, const UnstItems &I, unsigned long long c,
                                                             unsigned long long n_cand) {
    if (c >= n_cand) return I.tbase[I.n_items];
    const unsigned long long k = ui_item_of(I, c);
    uint32_t i, n;
    if (ui_kind(I, k, i, n) != UK_B) return I.tbase[k];
    const unsigned long long j = c - I.cbase[k];
    const uint32_t lo = I.lo[k];
    return I.tbase[k] + j * i + (U.lenpre[lo + j] - U.lenpre[lo]);
}

// One thread: the round that starts at candidate c0 ends at the largest c1 <= c0 + max_n whose text fits `cap` bytes, at
// least c0 + 1 (a candidate larger than a round is a round of its own).  uc->round = {c1, text bytes}.
__global__ void unstable_round_kernel(UnstTables U, UnstItems I, unsigned long long n_cand, unsigned long long c0,
                                      unsigned long long max_n, unsigned long long cap, UnstCounters *uc) {
    if (threadIdx.x | blockIdx.x) return;
    const unsigned long long base = ui_text_before(U, I, c0, n_cand);
    unsigned long long lo = c0 + 1, hi = min(n_cand, c0 + max_n);   // answer in [lo, hi]
    while (lo < hi) {
        const unsigned long long mid = (lo + hi + 1) >> 1;
        if (ui_text_before(U, I, mid, n_cand) - base <= cap) lo = mid; else hi = mid - 1;
    }
    uc->round[0] = lo;
    uc->round[1] = ui_text_before(U, I, lo, n_cand) - base;
}

// Is U[:i] + bytes(t) well-formed UTF-8?  U is; U[:i] may end inside a scalar that starts at b >= i - 3.  The junction
// U[b:i] + the leading continuation bytes of t goes through utf8_bad_word; the rest of t has a per-token flag.
__device__ __forceinline__ bool ut_utf8_join(const UnstTables &U, const uint8_t *u, uint32_t i, uint32_t t) {
    const uint8_t info = __ldg(U.u8info + t);
    if (!(info & 8u)) return false;
    const uint32_t c = info & 7u;
    uint32_t b = i;
    while (b > 0 && i - b < 3 && (u[b] & 0xC0u) == 0x80u) b--;
    if (b < i && (u[b] & 0xC0u) == 0x80u) return false;   // cannot happen in well-formed U
    if (b == i && c == 0) return true;
    if (c > 3) return false;
    uint8_t w[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint32_t n = 0;
    for (uint32_t k = b; k < i; k++) w[n++] = u[k];
    const uint8_t *tb = ut_bytes(U, t);
    for (uint32_t k = 0; k < c; k++) w[n++] = tb[k];
    const uint32_t zero[3] = {1u, 0u, 0u};               // one document that starts at byte 0
    return (utf8_bad_word(w, (int64_t)n, zero + 1, 0) & ((1u << n) - 1u)) == 0;
}

// Per candidate r of the round (c = c0 + r): cinfo = {doc, token, i, mode}; o_len[r] = its text in the ordinary run,
// s_len[2r], s_len[2r + 1] = its two documents in the single-piece run.
__global__ void __launch_bounds__(256) unstable_meta_kernel(UnstTables U, UnstItems I, const uint8_t *__restrict__ text,
                                                           unsigned long long c0, unsigned long long nr, uint4 *cinfo,
                                                           uint32_t *o_len, uint32_t *s_len, UnstCounters *uc) {
    const unsigned long long r = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (r >= nr) return;
    const unsigned long long c = c0 + r, k = ui_item_of(I, c);
    uint32_t i, n;
    const int kind = ui_kind(I, k, i, n);
    const uint32_t d = I.doc[k];
    const uint8_t *u = text + I.doc_off[d + 1] - n;
    uint32_t t = 0, mode, ol = 0, s0 = 0, s1 = 0;
    if (kind == UK_C) {
        uint32_t cp;
        s1 = ut_last_scalar(u, n, cp);
        s0 = n - s1;
        mode = UM_C;
    } else {
        t = __ldg(U.sorted + I.lo[k] + (uint32_t)(c - I.cbase[k]));
        if (kind == UK_A) mode = UM_A;
        else if (ut_utf8_join(U, u, i, t)) { mode = UM_ORD; ol = i + ut_len(U, t); }
        else { mode = UM_BPE; s0 = i + ut_len(U, t); }
    }
    cinfo[r] = make_uint4(d, t, i, mode);
    o_len[r] = ol; s_len[2 * r] = s0; s_len[2 * r + 1] = s1;
    const bool enc = mode != UM_A, bpe = mode >= UM_BPE;
    const unsigned m_enc = __ballot_sync(__activemask(), enc), m_bpe = __ballot_sync(__activemask(), bpe);
    if ((threadIdx.x & 31) == (unsigned)(__ffs(__activemask()) - 1)) {
        if (m_enc) atomicAdd(&uc->n_encoded, (unsigned long long)__popc(m_enc));
        if (m_bpe) atomicAdd(&uc->n_bpe, (unsigned long long)__popc(m_bpe));
    }
}

// One run's text: candidate r owns [off[r * stride], off[r * stride + stride]) and its bytes are U[:i] + bytes(t) (for
// (c): U).  16 output bytes per thread.
__global__ void __launch_bounds__(256) unstable_gather_kernel(UnstTables U, const uint8_t *__restrict__ text,
                                                             const unsigned long long *__restrict__ doc_off, const uint32_t *__restrict__ ulen,
                                                             const uint4 *__restrict__ cinfo, unsigned long long nr, int stride,
                                                             const unsigned long long *__restrict__ off, uint8_t *__restrict__ out) {
    const unsigned long long total = off[nr * stride];
    const unsigned long long q0 = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) * 16;
    if (q0 >= total) return;
    unsigned long long lo = 0, hi = nr;                 // off[lo * stride] <= q0 < off[hi * stride]
    while (hi - lo > 1) {
        const unsigned long long mid = (lo + hi) >> 1;
        if (off[mid * stride] <= q0) lo = mid; else hi = mid;
    }
    unsigned long long r = lo;
    const unsigned long long q1 = min(total, q0 + 16);
    for (unsigned long long q = q0; q < q1; q++) {
        while (off[(r + 1) * stride] <= q) r++;
        const uint4 ci = cinfo[r];
        const uint32_t n = ulen[ci.x], k = (uint32_t)(q - off[r * stride]);
        out[q] = k < ci.z ? text[doc_off[ci.x + 1] - n + k] : ut_bytes(U, ci.y)[k - ci.z];
    }
}

// The full token sequence of a round candidate, as two segments (each already replaced by the stored byte_pair_encode
// when it is one token its own merges do not reach).
struct CandSeq {
    const uint32_t *p0, *p1; uint32_t n0, n1;
    __device__ __forceinline__ uint32_t n() const { return n0 + n1; }
    __device__ __forceinline__ uint32_t at(uint32_t k) const { return k < n0 ? p0[k] : p1[k - n0]; }
};
struct RunOut {                 // run 2's outputs of the round
    const uint32_t *o_tok; const unsigned long long *o_off;     // ordinary run: candidate r = document r
    const uint32_t *s_tok; const unsigned long long *s_off;     // single-piece run: candidate r = documents 2r, 2r + 1
};
__device__ __forceinline__ void ut_bpe_seg(const UnstTables &U, const uint32_t *&p, uint32_t &n) {
    if (n == 1) {
        const uint32_t t = p[0];
        const uint32_t q = t < U.n_ids ? __ldg(U.ur_idx + t) : UR_NONE;
        if (q != UR_NONE) { p = U.ur_tok + __ldg(U.ur_off + q); n = __ldg(U.ur_off + q + 1) - __ldg(U.ur_off + q); }
    }
}
__device__ __forceinline__ CandSeq cand_seq(const UnstTables &U, const RunOut &R, const uint4 *cinfo, unsigned long long r) {
    CandSeq s;
    const uint32_t mode = cinfo[r].w;
    s.p1 = nullptr; s.n1 = 0;
    if (mode == UM_A) { s.p0 = &cinfo[r].y; s.n0 = 1; }
    else if (mode == UM_ORD) { s.p0 = R.o_tok + R.o_off[r]; s.n0 = (uint32_t)(R.o_off[r + 1] - R.o_off[r]); }
    else {
        s.p0 = R.s_tok + R.s_off[2 * r]; s.n0 = (uint32_t)(R.s_off[2 * r + 1] - R.s_off[2 * r]);
        s.p1 = R.s_tok + R.s_off[2 * r + 1]; s.n1 = (uint32_t)(R.s_off[2 * r + 2] - R.s_off[2 * r + 1]);
        ut_bpe_seg(U, s.p0, s.n0);
        ut_bpe_seg(U, s.p1, s.n1);
    }
    return s;
}

struct UnstTable {              // open addressing over (document, completion); key 0 = empty
    unsigned long long *key; uint32_t *idx; uint32_t *loc; uint32_t mask;
};
struct UnstResult {             // a chunk's distinct completions so far
    uint32_t *tok; unsigned long long *off; uint32_t *doc; uint32_t *grp;
};

// Per candidate: tokens kept (up to the first at which the byte count reaches |U|, lib.rs:574-582), their key, its slot.
__global__ void __launch_bounds__(256) unstable_insert_kernel(UnstTables U, RunOut R, const uint4 *__restrict__ cinfo,
                                                             const uint32_t *__restrict__ ulen, unsigned long long c0,
                                                             unsigned long long nr, unsigned long long seed, UnstTable H,
                                                             uint32_t *nkeep, uint32_t *slot, UnstCounters *uc, Counters *ctr) {
    const unsigned long long r = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (r >= nr) return;
    const CandSeq s = cand_seq(U, R, cinfo, r);
    const uint32_t d = cinfo[r].x, need = ulen[d];
    uint32_t acc = 0, k = 0;
    unsigned long long h = long_hash_init(seed ^ d);
    while (k < s.n()) {
        const uint32_t t = s.at(k);
        if (t >= PSEUDO_BASE) { atomicOr(&ctr->err, ERR_NOBYTE); break; }   // a stored byte_pair_encode needs a missing byte
        h = long_hash_step(h, t, k);
        k++;
        acc += ut_len(U, t);
        if (acc >= need) break;
    }
    nkeep[r] = k;
    unsigned long long key = (long_hash_word(h, d) ^ seed) | 1ull;
    uint32_t s0 = (uint32_t)(key ^ (key >> 32)) & H.mask;
    for (int p = 0; p < UNST_PROBES; p++, s0 = (s0 + 1) & H.mask) {
        const unsigned long long old = atomicCAS(&H.key[s0], 0ull, key);
        if (old == 0ull || old == key) {
            atomicMin(&H.idx[s0], (uint32_t)(c0 + r));
            slot[r] = s0;
            return;
        }
    }
    slot[r] = 0xFFFFFFFFu;
    atomicOr(&uc->err, UERR_TABLE);
}

// Per candidate: keep[r] = 1 when it is the first occurrence of its (document, completion); kc[r] = its tokens then.
__global__ void __launch_bounds__(256) unstable_verify_kernel(UnstTables U, RunOut R, const uint4 *__restrict__ cinfo,
                                                             unsigned long long c0, unsigned long long nr, UnstTable H,
                                                             UnstResult res, const uint32_t *__restrict__ nkeep,
                                                             const uint32_t *__restrict__ slot, uint32_t *keep, uint32_t *kc,
                                                             UnstCounters *uc) {
    const unsigned long long r = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (r >= nr) return;
    const uint32_t sl = slot[r];
    uint32_t kp = 0;
    if (sl != 0xFFFFFFFFu) {
        const uint32_t m = H.idx[sl], c = (uint32_t)(c0 + r), n = nkeep[r];
        if (m == c) kp = 1;
        else {
            const CandSeq s = cand_seq(U, R, cinfo, r);
            bool same;
            if (m < c0) {                                // the winner is a completion of an earlier round
                const uint32_t q = H.loc[sl];
                const unsigned long long a = res.off[q];
                same = res.doc[q] == cinfo[r].x && res.off[q + 1] - a == n;
                for (uint32_t k = 0; same && k < n; k++) same = res.tok[a + k] == s.at(k);
            } else {
                const unsigned long long rm = m - c0;
                const CandSeq w = cand_seq(U, R, cinfo, rm);
                same = cinfo[rm].x == cinfo[r].x && nkeep[rm] == n;
                for (uint32_t k = 0; same && k < n; k++) same = w.at(k) == s.at(k);
            }
            if (!same) atomicOr(&uc->err, UERR_COLLIDE);
        }
    }
    keep[r] = kp;
    kc[r] = kp ? nkeep[r] : 0u;
}

// The kept candidates, in candidate order: completion q = n_comp + cbase[r] at token offset n_tok + tbase[r].
__global__ void __launch_bounds__(256) unstable_write_kernel(UnstTables U, RunOut R, const uint4 *__restrict__ cinfo,
                                                            unsigned long long nr, UnstTable H, UnstResult res,
                                                            const uint32_t *__restrict__ keep, const uint32_t *__restrict__ kc,
                                                            const uint32_t *__restrict__ slot,
                                                            const unsigned long long *__restrict__ cbase,
                                                            const unsigned long long *__restrict__ tbase,
                                                            unsigned long long n_comp, unsigned long long n_tok) {
    const unsigned long long r = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (r >= nr || !keep[r]) return;
    const CandSeq s = cand_seq(U, R, cinfo, r);
    const unsigned long long q = n_comp + cbase[r], a = n_tok + tbase[r];
    const uint32_t n = kc[r];
    for (uint32_t k = 0; k < n; k++) res.tok[a + k] = s.at(k);
    res.off[q] = a;
    if (cbase[r] + 1 == cbase[nr]) res.off[q + 1] = a + n;   // the end of the last completion so far (later rounds compare with it)
    res.doc[q] = cinfo[r].x;
    H.loc[slot[r]] = (uint32_t)q;
    atomicAdd(&res.grp[cinfo[r].x], 1u);
}
