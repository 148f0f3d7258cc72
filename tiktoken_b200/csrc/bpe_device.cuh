// bpe_device.cuh -- table layouts, hashing and the per-thread BPE merge shared by the CUDA kernels
// (and, through hostcheck.cpp, by the CPU-only unit tests of exactly this code).
//
// Reference being replaced: the byte-slice -> rank FxHashMap probes and the min-rank merge loop
// of src/lib.rs:140-211 (`_byte_pair_merge`, `byte_pair_encode`) and the whole-piece probe of
// src/lib.rs:367-368.
//
// Design (see DESIGN.md):
//  * token id == rank.  A single byte the vocabulary lacks gets a pseudo id PSEUDO_BASE+byte so
//    that merges through it still work; emitting one is the reference's panic (lib.rs:202,207).
//  * PIECE tables: open-addressed, keyed by the piece bytes themselves -> exact compare.  Tokens of
//    1..11 bytes go to the NARROW table, one 16-byte slot per probe step (key words + length + rank);
//    tokens of 12..16 bytes to the WIDE table, 32-byte slots (key words, then length + rank).
//  * LONG-token table: tokens > 16 bytes, keyed by a 64-bit hash, verified against a byte blob.
//  * PAIR table: (id(A), id(B)) -> rank(A||B) for every split of every token into two parts that
//    are themselves tokens (or single bytes).  Because every part produced by the merge loop is
//    a token, probing bytes(A)||bytes(B) in the reference's map is the same as probing
//    (id(A), id(B)) here -- fixed 8-byte keys, no variable-length hashing inside the loop
//    (the reference's own remark, lib.rs:145-147 and :259-260).  16-byte slots, probed one at a time.
//  * PAIR2: direct 64 Ki-entry table for the initial byte pairs (lib.rs:149-155).
#pragma once
#include <stdint.h>
#include "pretok_rules.cuh"

namespace b2bpe {

static const uint32_t RANK_MAX = 0xFFFFFFFFu;
static const uint32_t PSEUDO_BASE = 0xFFFFFE00u;   // ids >= this are "byte missing from vocabulary"
static const int SHORT_MAX = 16;                   // pieces up to this length take the per-thread path
static const uint32_t NARROW_MAX = 11;             // tokens up to this length live in the narrow piece table
static const uint32_t PAIR_EMPTY = 0xFFFFFFFFu;    // `a` of an empty pair-table slot (no token id is this large)
static const uint32_t PIECE_THROUGH = 0x80000000u; // pass-through mark in the rank word of a narrow piece slot

struct U4 { uint32_t x, y, z, w; };                // host mirror of uint4

struct DevTables {
    const uint32_t *byte_id;      // [256]
    const uint32_t *pair2;        // [65536] rank of the 2-byte token b0,b1 (index b0*256+b1) or RANK_MAX
    const U4 *pair_tab;           // one slot {a, b, rank, through} per probe step; empty slot: a == PAIR_EMPTY, through == 0
    uint32_t pair_mask;           // number of slots - 1
    const U4 *narrow_tab;         // tokens of 1..11 bytes, one U4 per slot: {w0, w1, w2 | len << 24, rank | through << 31}; empty: 0
    uint32_t narrow_mask;
    const U4 *wide_tab;           // tokens of 12..16 bytes, 2 x U4 per slot: {w0, w1, w2, w3} {len, rank, through, 0}; empty: 0
    uint32_t wide_mask;
    const U4 *long_tab;           // 2 x U4 per slot: {hlo, hhi, blob_off, len} {rank,0,0,0}; empty: len == 0
    uint32_t long_mask;
    const uint8_t *long_blob;
    uint32_t max_token_len;
    uint32_t n_long_tokens;
};

#if defined(__CUDA_ARCH__)
#define B2_LDG_U4(p) b2bpe::ldg_u4(p)
#define B2_LDG_U32(p) __ldg(p)
__device__ __forceinline__ U4 ldg_u4(const U4 *p) {
    uint4 v = __ldg(reinterpret_cast<const uint4 *>(p));
    U4 r; r.x = v.x; r.y = v.y; r.z = v.z; r.w = v.w; return r;
}
#else
#define B2_LDG_U4(p) (*(p))
#define B2_LDG_U32(p) (*(p))
#endif

B2_HD uint32_t pair_hash(uint32_t a, uint32_t b) {
    uint32_t h = a * 0x9E3779B1u;
    h ^= (b + 0x7F4A7C15u) * 0x85EBCA6Bu;
    h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 13;
    return h;
}

// Hash of a piece of <= 16 bytes given as four little-endian words (zero padded) + its length: 32-bit
// multiply-xorshift rounds (one IMAD per word), not a 64-bit mix -- the probe kernel hashes every piece of the
// corpus, and 64-bit multiplies are four instructions each on the SM.
B2_HD uint32_t piece_hash4(uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t len) {
    uint32_t h = (a0 ^ (len * 0x9E3779B1u)) * 0x85EBCA6Bu;
    h ^= h >> 13;
    h = (h ^ a1) * 0xC2B2AE35u;
    h ^= h >> 16;
    h = (h ^ a2) * 0x27D4EB2Fu;
    h ^= h >> 15;
    h = (h ^ a3) * 0x165667B1u;
    h ^= h >> 16;
    return h;
}
B2_HD uint32_t piece_hash(uint64_t k0, uint64_t k1, uint32_t len) {
    return piece_hash4((uint32_t)k0, (uint32_t)(k0 >> 32), (uint32_t)k1, (uint32_t)(k1 >> 32), len);
}

// 64-bit hash of a byte string given as little-endian u64 words (last one zero padded):
// init(len) XOR the mixes of (word, index) -- order-independent, so a warp hashes a piece with one
// word per lane and an XOR reduction.
B2_HD uint64_t long_hash_word(uint64_t w, uint32_t i) {
    uint64_t x = (w ^ ((uint64_t)(i + 1) * 0x9E3779B97F4A7C15ull)) * 0xC2B2AE3D27D4EB4Full;
    x ^= x >> 29; x *= 0x165667B19E3779F9ull;
    return x ^ (x >> 32);
}
B2_HD uint64_t long_hash_step(uint64_t h, uint64_t w, uint32_t i) { return h ^ long_hash_word(w, i); }
B2_HD uint64_t long_hash_init(uint64_t len) { return len * 0xC2B2AE3D27D4EB4Full + 0x165667B19E3779F9ull; }

// ---- miss memo key: the zero-padded bytes of a missed piece of 1..15 bytes with its length in byte 15 ------------------
// Bytes len..14 are zero and byte 15 is the length, so equal keys mean equal (bytes, length), NUL bytes included, and no
// key is all zero (an empty memo slot).  A 16-byte piece has no spare byte: it is not memoised (false).
B2_HD bool memo_key(U4 &k, uint32_t len) {
    if (len >= (uint32_t)SHORT_MAX) return false;
    k.w |= len << 24;
    return true;
}
B2_HD uint32_t memo_hash(const U4 &k) {
    const uint64_t lo = ((uint64_t)k.y << 32 | k.x), hi = ((uint64_t)k.w << 32 | k.z);
    return (uint32_t)(long_hash_word(lo, 0) ^ long_hash_word(hi, 1));
}

// ---- pair table: linear probing over 16-byte slots {a, b, rank, through} ----------------------------------------
// `through` is 1 when the probe path of some key passes the slot (bpe_tables.h): a slot that does not hold the key and is
// not passed through -- an empty slot included -- ends the chain.
// A probe is its start position, then steps: load the slot at s (pair_slot), look at it (pair_step).  Callers with
// several probes load all their slots before they look at any, so the loads are in flight together.
B2_HD uint32_t pair_start(const DevTables &T, uint32_t a, uint32_t b) { return pair_hash(a, b) & T.pair_mask; }
B2_HD U4 pair_slot(const DevTables &T, uint32_t s) { return B2_LDG_U4(T.pair_tab + s); }
// one probe step on the slot e loaded from position s: true when the chain ends (r = the rank, or RANK_MAX for an
// absent pair), otherwise s moves to the next slot
B2_HD bool pair_step(const DevTables &T, const U4 &e, uint32_t a, uint32_t b, uint32_t &s, uint32_t &r) {
    if (e.x == a && e.y == b) { r = e.z; return true; }
    if (e.w == 0) { r = RANK_MAX; return true; }
    s = (s + 1) & T.pair_mask;
    return false;
}

B2_HD uint32_t pair_lookup(const DevTables &T, uint32_t a, uint32_t b) {
    uint32_t s = pair_start(T, a, b), r = RANK_MAX;
    while (!pair_step(T, pair_slot(T, s), a, b, s, r)) {}
    return r;
}

// two independent pair probes with both first loads in flight together (the two neighbours of a
// merge, src/lib.rs:182-185)
B2_HD void pair_lookup2(const DevTables &T, uint32_t a1, uint32_t b1, uint32_t a2, uint32_t b2, uint32_t &r1,
                        uint32_t &r2) {
    uint32_t s1 = pair_start(T, a1, b1), s2 = pair_start(T, a2, b2);
    const U4 e1 = pair_slot(T, s1), e2 = pair_slot(T, s2);
    if (!pair_step(T, e1, a1, b1, s1, r1)) while (!pair_step(T, pair_slot(T, s1), a1, b1, s1, r1)) {}
    if (!pair_step(T, e2, a2, b2, s2, r2)) while (!pair_step(T, pair_slot(T, s2), a2, b2, s2, r2)) {}
}

// ---- piece tables: whole-piece probe for len <= 16 (src/lib.rs:367-368) ---------------------------------------
// The key is the piece as four little-endian words a0..a3, zero padded beyond len.  The table depends on len only: a
// narrow piece (len <= 11: byte 11 of its key is padding and carries len in the slot) loads one 16-byte slot per step, a
// wide one both halves of a 32-byte slot.  As in the pair table, a slot carries a pass-through mark (bit 31 of a narrow
// slot's rank word -- ranks are < 2^30 --, word z of a wide slot's second half): a slot that does not hold the key and is
// not passed through ends the chain.  A probe is issued (first slot loaded) and finished (compare, continue the chain)
// separately, so that a caller can keep several probes in flight.
B2_HD void piece_load(const DevTables &T, uint32_t len, uint32_t s, U4 &e0, U4 &e1) {
    const bool narrow = len <= NARROW_MAX;
    const U4 *p = narrow ? T.narrow_tab + s : T.wide_tab + 2 * s;
    e0 = B2_LDG_U4(p);
    if (!narrow) e1 = B2_LDG_U4(p + 1);                      // e1 is not looked at for a narrow piece
}
// returns the probe position; e0 / e1 receive the slot there
B2_HD uint32_t piece_issue(const DevTables &T, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t len,
                           U4 &e0, U4 &e1) {
    const uint32_t s = piece_hash4(a0, a1, a2, a3, len) & (len <= NARROW_MAX ? T.narrow_mask : T.wide_mask);
    piece_load(T, len, s, e0, e1);
    return s;
}
// the rank of the piece, or RANK_MAX; e0 / e1 is the slot at s that piece_issue loaded
B2_HD uint32_t piece_finish(const DevTables &T, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t len,
                            uint32_t s, U4 e0, U4 e1) {
    const bool narrow = len <= NARROW_MAX;
    const uint32_t mask = narrow ? T.narrow_mask : T.wide_mask;
    const uint32_t z = narrow ? (a2 | len << 24) : a2;
    for (;;) {
        if (e0.x == a0 && e0.y == a1 && e0.z == z && (narrow || (e0.w == a3 && e1.x == len)))
            return narrow ? e0.w & ~PIECE_THROUGH : e1.y;
        if ((narrow ? e0.w & PIECE_THROUGH : e1.z) == 0) return RANK_MAX;   // no chain passes here (empty slots included)
        s = (s + 1) & mask;
        piece_load(T, len, s, e0, e1);
    }
}
B2_HD uint32_t piece_lookup16(const DevTables &T, uint64_t k0, uint64_t k1, uint32_t len) {
    const uint32_t a0 = (uint32_t)k0, a1 = (uint32_t)(k0 >> 32), a2 = (uint32_t)k1, a3 = (uint32_t)(k1 >> 32);
    U4 e0 = {0, 0, 0, 0}, e1 = {0, 0, 0, 0};
    const uint32_t s = piece_issue(T, a0, a1, a2, a3, len, e0, e1);
    return piece_finish(T, a0, a1, a2, a3, len, s, e0, e1);
}

// whole-piece probe for len > 16: hash already computed; bytes compared against the blob
template <class ByteFn>
B2_HD uint32_t piece_lookup_long(const DevTables &T, uint64_t h, uint32_t len, ByteFn byte_at) {
    if (T.n_long_tokens == 0 || len > T.max_token_len) return RANK_MAX;
    uint32_t s = (uint32_t)(h ^ (h >> 32)) & T.long_mask;
    for (;;) {
        U4 k = B2_LDG_U4(T.long_tab + 2 * s);
        if (k.w == 0) return RANK_MAX;
        if (k.w == len && k.x == (uint32_t)h && k.y == (uint32_t)(h >> 32)) {
            const uint8_t *ref = T.long_blob + k.z;
            bool same = true;
            for (uint32_t i = 0; i < len; i++) if (ref[i] != byte_at(i)) { same = false; break; }
            if (same) return B2_LDG_U4(T.long_tab + 2 * s + 1).x;
        }
        s = (s + 1) & T.long_mask;
    }
}

B2_HD int b2_ffs(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __ffs((int)x);
#else
    return __builtin_ffs((int)x);
#endif
}
B2_HD int b2_clz(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __clz((int)x);
#else
    return x ? __builtin_clz(x) : 32;
#endif
}

// ------------------------------------------------------------------------------------------
// Per-thread merge for a piece of 2..16 bytes: the literal loop of `_byte_pair_merge`
// (src/lib.rs:140-196): repeatedly merge the adjacent pair of smallest rank, leftmost on ties
// (strict `<`, lib.rs:151 / :190), until no adjacent pair is a token.  Parts are a bit mask of
// start offsets; id[j] / rk[j] hold the part starting at j and the rank of (part j, next part).
// IdArr / RkArr are per-thread views (a shared-memory column on the device, plain arrays on the
// host).  Returns the mask of token start offsets; token ids are id[j] at the set bits.
// ------------------------------------------------------------------------------------------
template <class ByteFn, class IdArr, class RkArr>
B2_HD uint32_t merge_short(const DevTables &T, ByteFn byte_at, int n, IdArr id, RkArr rk) {
    uint32_t prevb = byte_at(0);
    for (int j = 0; j < n; j++) {
        uint32_t nb = (j + 1 < n) ? byte_at(j + 1) : 0;
        id[j] = B2_LDG_U32(T.byte_id + prevb);
        rk[j] = (j + 1 < n) ? B2_LDG_U32(T.pair2 + (prevb << 8 | nb)) : RANK_MAX;
        prevb = nb;
    }
    uint32_t mask = (n >= 32) ? 0xFFFFFFFFu : ((1u << n) - 1u);
    for (;;) {
        uint32_t best = RANK_MAX; int bj = -1;
        for (uint32_t m = mask; m;) {
            int j = b2_ffs(m) - 1; m &= m - 1;
            uint32_t r = rk[j];
            if (r < best) { best = r; bj = j; }
        }
        if (best == RANK_MAX) break;
        uint32_t above = mask & ~((2u << bj) - 1u);
        int j2 = b2_ffs(above) - 1;                 // right part of the merged pair
        mask &= ~(1u << j2);
        id[bj] = best;                              // id == rank of the merged token
        above &= ~(1u << j2);
        const uint32_t below = mask & ((1u << bj) - 1u);
        if (above && below) {
            const int jp = 31 - b2_clz(below);
            uint32_t rr, rl;
            pair_lookup2(T, best, id[b2_ffs(above) - 1], id[jp], best, rr, rl);
            rk[bj] = rr; rk[jp] = rl;
        } else if (above) {
            rk[bj] = pair_lookup(T, best, id[b2_ffs(above) - 1]);
        } else {
            rk[bj] = RANK_MAX;
            if (below) { const int jp = 31 - b2_clz(below); rk[jp] = pair_lookup(T, id[jp], best); }
        }
    }
    return mask;
}

// ------------------------------------------------------------------------------------------
// Warp-convergent form of merge_short for the encode kernel: every lane of `group` (a lane mask)
// merges its own piece, but all lanes walk the SAME instruction stream -- fixed trip counts
// (n_max = longest piece in the group), selects instead of data-dependent branches -- so the
// warp issues one stream per round instead of one per lane.  Same result as merge_short
// (hostcheck runs both against the oracle).  A lane with n == 0 just idles along.
// ------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
#define B2_ANY(group, pred) __any_sync(group, pred)
#else
#define B2_ANY(group, pred) (pred)
#endif

template <int MAXN = 16, class ByteFn, class IdArr, class RkArr>
B2_HD uint32_t merge_short_conv(const DevTables &T, ByteFn byte_at, int n, int n_max, unsigned group,
                                IdArr id, RkArr rk) {
#if defined(__CUDA_ARCH__)
    // initial ids / pair ranks, 16 parts at a time: all table loads of a block are issued before the first store
    // waits for one (a rolled loop serialises one L2 round trip per part)
#pragma unroll
    for (int h = 0; h < MAXN; h += 16) {
        if (h < n_max) {
            uint32_t iv[16], rv[16];
#pragma unroll
            for (int k = 0; k < 16; k++) {
                const int j = h + k;
                iv[k] = 0; rv[k] = RANK_MAX;
                if (j < n) {
                    const uint32_t b0 = byte_at(j);
                    iv[k] = B2_LDG_U32(T.byte_id + b0);
                    if (j + 1 < n) rv[k] = B2_LDG_U32(T.pair2 + (b0 << 8 | byte_at(j + 1)));
                }
            }
#pragma unroll
            for (int k = 0; k < 16; k++)
                if (h + k < n_max) { id[h + k] = iv[k]; rk[h + k] = rv[k]; }
        }
    }
#else
    for (int j = 0; j < n_max; j++) {
        uint32_t i0 = 0, r0 = RANK_MAX;
        if (j < n) {
            const uint32_t b0 = byte_at(j);
            i0 = B2_LDG_U32(T.byte_id + b0);
            if (j + 1 < n) r0 = B2_LDG_U32(T.pair2 + (b0 << 8 | byte_at(j + 1)));
        }
        id[j] = i0; rk[j] = r0;
    }
#endif
    uint32_t mask = n <= 0 ? 0u : ((n >= 32) ? 0xFFFFFFFFu : ((1u << n) - 1u));
    for (;;) {
        uint32_t best = RANK_MAX; int bj = 0;
        for (int j = 0; j < n_max; j++) {                      // dead / absent parts hold RANK_MAX
            const uint32_t r = rk[j];
            const bool lt = r < best;
            best = lt ? r : best; bj = lt ? j : bj;
        }
        const bool act = best != RANK_MAX;
        if (!B2_ANY(group, act)) break;
        uint32_t a1 = 0, b1 = 0, a2 = 0, b2 = 0; bool need_r = false, need_l = false; int jp = 0;
        if (act) {
            uint32_t above = mask & ~((2u << bj) - 1u);
            const int j2 = b2_ffs(above) - 1;
            mask &= ~(1u << j2);
            rk[j2] = RANK_MAX;                                 // the right part disappears
            id[bj] = best;
            above &= ~(1u << j2);
            const uint32_t below = mask & ((1u << bj) - 1u);
            if (above) { need_r = true; a1 = best; b1 = id[b2_ffs(above) - 1]; }
            if (below) { need_l = true; jp = 31 - b2_clz(below); a2 = id[jp]; b2 = best; }
        }
        // the two neighbour probes of every active lane, issued together
        uint32_t s1 = pair_start(T, a1, b1), s2 = pair_start(T, a2, b2);
        uint32_t r1 = RANK_MAX, r2 = RANK_MAX;
        bool p1 = need_r, p2 = need_l;
        while (B2_ANY(group, p1 || p2)) {
            U4 e = {0, 0, 0, 0}, f = {0, 0, 0, 0};
            if (p1) e = pair_slot(T, s1);
            if (p2) f = pair_slot(T, s2);
            if (p1) p1 = !pair_step(T, e, a1, b1, s1, r1);
            if (p2) p2 = !pair_step(T, f, a2, b2, s2, r2);
        }
        if (act) {
            rk[bj] = need_r ? r1 : RANK_MAX;
            if (need_l) rk[jp] = r2;
        }
    }
    return mask;
}

// ------------------------------------------------------------------------------------------
// Thread-per-piece merge for MID-size pieces (17 .. a few hundred bytes), warp-convergent like
// merge_short_conv: every lane of `group` owns one piece and all lanes walk one instruction
// stream (n_max = longest piece in the group).  The literal loop of `_byte_pair_merge`
// (src/lib.rs:140-196): take the smallest rank (strict `<` => leftmost on ties), merge, re-rank
// the two neighbouring pairs.
// Parts live in two per-lane columns.  For the part that STARTS at byte j: id[j] = its token id,
// rk[j] = rank of (part j, next part) or RANK_MAX.  A byte absorbed by the part to its left is DEAD:
// id[j] = ID_DEAD and rk[j] is free, so the first and the last dead byte of every part carry a link
// word MID_LINK | start << 12 | len of that part -- the neighbours of a part are found with two loads
// instead of a walk over dead bytes.  Link words (and RANK_MAX) compare above every rank (< 2^30).
// The minimum is kept two-level: gmin[g] / gpos[g] = smallest rank (leftmost) of the MID_G entries
// of group g, so a round scans n / MID_G group minima and re-scans only the three groups whose
// entries changed.  On return the tokens are the live id[j], j < n, left to right.
// ------------------------------------------------------------------------------------------
static const uint32_t ID_DEAD = 0xFFFFFFFFu;
static const uint32_t MID_LINK = 0x80000000u;
static const uint32_t MID_NONE = 0x40000000u;                  // "no mergeable pair": above every rank
static const int MID_G = 8;

template <class RkArr>
B2_HD void mid_group_min(RkArr rk, int g, uint32_t &best, uint32_t &pos) {
    best = MID_NONE; int bj = 0;
#pragma unroll
    for (int k = 0; k < MID_G; k++) {
        const uint32_t r = rk[g * MID_G + k];
        const bool lt = r < best;
        best = lt ? r : best; bj = lt ? k : bj;
    }
    pos = (uint32_t)(g * MID_G + bj);
}

// id / rk need MID_G * ceil(n_max / MID_G) entries, gmin / gpos ceil(n_max / MID_G).
// On entry rk[0 .. n_max) holds the piece's BYTES (the caller stages them; it needs them for the whole-piece
// probe anyway), so that no pass here carries a dependent global-load chain.
template <class IdArr, class RkArr, class GArr>
B2_HD void merge_mid_conv(const DevTables &T, int n, int n_max, unsigned group, IdArr id, RkArr rk, GArr gmin, GArr gpos) {
    const int ng = (n_max + MID_G - 1) / MID_G;
    {
        for (int j = n_max; j < ng * MID_G; j++) rk[j] = 0u;
#pragma unroll 4
        for (int j = 0; j < ng * MID_G; j++) {
            const uint32_t b0 = rk[j], b1 = (j + 1 < ng * MID_G) ? rk[j + 1] : 0u;
            uint32_t i0 = ID_DEAD, r0 = RANK_MAX;
            if (j < n) {
                i0 = B2_LDG_U32(T.byte_id + b0);
                if (j + 1 < n) r0 = B2_LDG_U32(T.pair2 + (b0 << 8 | b1));
            }
            id[j] = i0; rk[j] = r0;
        }
        for (int g = 0; g < ng; g++) { uint32_t m, q; mid_group_min(rk, g, m, q); gmin[g] = m; gpos[g] = q; }
    }
    const int half = (ng + 1) >> 1;
    for (;;) {
        // two independent chains over the group minima (left half / right half); the right half wins
        // only when strictly smaller => leftmost on ties
        uint32_t bestA = MID_NONE, bestB = MID_NONE; int gA = 0, gB = 0;
        for (int g = 0; g < half; g++) {
            const uint32_t ra = gmin[g];
            const uint32_t rb = (g + half < ng) ? gmin[g + half] : MID_NONE;
            const bool la = ra < bestA, lb = rb < bestB;
            bestA = la ? ra : bestA; gA = la ? g : gA;
            bestB = lb ? rb : bestB; gB = lb ? g + half : gB;
        }
        const uint32_t best = bestB < bestA ? bestB : bestA;
        const int bg = bestB < bestA ? gB : gA;
        const bool act = best < MID_NONE;
        if (!B2_ANY(group, act)) break;
        int bj = 0, j2 = 1, j3 = n, jp = -1;
        if (act) {
            bj = (int)gpos[bg];
            j2 = bj + 1; jp = bj - 1;
            // right part of the merged pair (exists: rk[bj] is the rank of (bj, next)), the part after it
            // and the left neighbour -- via the link words of the dead bytes at the parts' ends
            if (id[j2] == ID_DEAD) j2 = bj + (int)(rk[j2] & 0xFFFu);
            j3 = j2 + 1;
            if (j3 < n && id[j3] == ID_DEAD) j3 = j2 + (int)(rk[j3] & 0xFFFu);
            if (jp >= 0 && id[jp] == ID_DEAD) jp = (int)((rk[jp] >> 12) & 0xFFFu);
        }
        const bool need_r = act && j3 < n, need_l = act && jp >= 0;
        uint32_t a1 = 0, b1 = 0, a2 = 0, b2 = 0;
        if (need_r) { a1 = best; b1 = id[j3]; }
        if (need_l) { a2 = id[jp]; b2 = best; }
        if (act) {
            const uint32_t link = MID_LINK | ((uint32_t)bj << 12) | (uint32_t)(j3 - bj);
            id[bj] = best; id[j2] = ID_DEAD;
            rk[j2] = link; rk[bj + 1] = link; rk[j3 - 1] = link;
        }
        // the two neighbour probes of every active lane, issued together
        uint32_t s1 = pair_start(T, a1, b1), s2 = pair_start(T, a2, b2);
        uint32_t r1 = RANK_MAX, r2 = RANK_MAX;
        bool p1 = need_r, p2 = need_l;
        while (B2_ANY(group, p1 || p2)) {
            U4 e = {0, 0, 0, 0}, f = {0, 0, 0, 0};
            if (p1) e = pair_slot(T, s1);
            if (p2) f = pair_slot(T, s2);
            if (p1) p1 = !pair_step(T, e, a1, b1, s1, r1);
            if (p2) p2 = !pair_step(T, f, a2, b2, s2, r2);
        }
        if (act) {
            rk[bj] = need_r ? r1 : RANK_MAX;
            if (need_l) rk[jp] = r2;
            // the groups whose ranks changed: bj's, j2's (its rank became a link) and jp's; duplicates
            // just recompute the same values, so the three scans run back to back without votes
            const int g1 = bj / MID_G, g2 = j2 / MID_G, g0 = need_l ? jp / MID_G : g1;
            uint32_t m0, q0, m1, q1, m2, q2;
            mid_group_min(rk, g0, m0, q0); mid_group_min(rk, g1, m1, q1); mid_group_min(rk, g2, m2, q2);
            gmin[g0] = m0; gpos[g0] = q0; gmin[g1] = m1; gpos[g1] = q1; gmin[g2] = m2; gpos[g2] = q2;
        }
    }
}

}  // namespace b2bpe
