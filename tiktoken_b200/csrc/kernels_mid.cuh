// kernels_mid.cuh -- pieces of 17..1024 bytes (CJK runs, indentation, separators, long identifiers, digit runs): a
// GROUP OF LANES per piece.  The literal loop of `_byte_pair_merge` (src/lib.rs:140-196): take the smallest rank
// (strict `<` => leftmost on ties), merge, re-rank the two neighbouring pairs -- one merge per round.
//
// The cost of this stage is the number of warp instructions per merge round, so the layout is
// chosen to (a) share one instruction stream between as many pieces as possible and (b) keep a round short:
//   * a piece of up to G*E bytes is spread over G lanes, E parts per lane (G x E = 2x16, 4x16, 4x32, 8x32, 32x32 for
//     the classes 17-32, 33-64, 65-128, 129-256, 257-1024 bytes): 32 / G pieces walk one convergent instruction stream;
//   * every lane takes the minimum of its own E keys (E independent shared loads), the group minimum is a log2(G)-step
//     shuffle butterfly -- keys are (rank << 10 | position), so the minimum IS the leftmost smallest rank;
//   * the neighbours of the merged pair come from a doubly linked list of live parts in shared memory (one packed word
//     per part: next | prev << 16): three loads, two stores per round, no walk over dead bytes;
//   * the two pair-table probes of a round run on two different lanes at the same time.
// The state of a warp is (key + id + link) x E x 32 words of shared memory whatever the class, and warps are
// independent (no block barriers): a warp steps through its classes on its own.
// Keys pack the rank into 22 bits: vocabularies with ranks of 2^22 and above keep using the lane-per-piece and
// warp-per-piece kernels of kernels_long.cuh.
#pragma once
#include "dev_common.cuh"

using namespace b2bpe;

static const int MIDG_WARPS = 4;                 // warps per block (independent of each other)
static const uint32_t MIDG_NONE = 0xFFFFFFFFu;   // "no mergeable pair here" (above every key)
static const uint32_t MIDG_NIL = 0xFFFFu;        // end of the part list
static const int MIDG_POS_BITS = 10;
static const uint32_t MIDG_MAX_RANK = 1u << (32 - MIDG_POS_BITS);

template <int E>
struct MidGSmem {
    uint32_t key[E * 32];                        // [slot][lane]: rank of (this part, next part) << 10 | position, or MIDG_NONE
    uint32_t id[E * 32];                         // [slot][lane]: token id of the part that starts here
    uint32_t link[E * 32];                       // [slot][lane]: position of the next live part | previous one << 16
};

template <int G, int E>
__device__ void midg_class(const uint8_t *__restrict__ text, const DevTables &T, const LongQ &q, int cls, uint32_t *ltok,
                           Counters *ctr, MidGSmem<E> &S) {
    static_assert(E == 16 || E == 32, "parts per lane");
    constexpr int LOG_E = E == 16 ? 4 : 5;
    constexpr int P = 32 / G;                    // pieces per warp pass
    constexpr int NW = E / 8;                    // 64-bit words of piece bytes per lane
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);               // lane within the group
    const int gb = lane & ~(G - 1);              // first lane of the group
    const unsigned int n_items = ctr->n_cls[cls];
    const unsigned int *list = q.cls[cls];
    uint32_t *const keyc = S.key + lane, *const idc = S.id + lane, *const linkc = S.link + lane;   // this lane's columns: [slot * 32]
    // shared-memory index of the part at position j of this lane's group
    auto at = [&](uint32_t j) -> uint32_t { return (j & (E - 1)) * 32u + (uint32_t)gb + (j >> LOG_E); };
    for (;;) {
        unsigned int k0 = 0;
        if (lane == 0) k0 = atomicAdd(&ctr->cls_head[cls], (unsigned int)P);
        k0 = __shfl_sync(0xFFFFFFFFu, k0, 0);
        if (k0 >= n_items) break;
        const unsigned int item = k0 + (unsigned int)(lane / G);
        const bool have = item < n_items;
        unsigned int qi = 0; unsigned long long st = 0; int n = 0;
        if (have) { qi = list[item]; st = q.start[qi]; n = (int)q.len[qi]; }
        const uint8_t *piece = text + st;
        uint32_t *out = ltok + st;
        // ---- this lane's E bytes (+ the first byte of the next lane's), packed in 64-bit words ----------------
        const int j0 = gl * E;
        uint64_t w[NW]; uint32_t bnext = 0;
#pragma unroll
        for (int k = 0; k < NW; k++) {
            w[k] = 0;
#pragma unroll
            for (int s = 0; s < 8; s++)
                if (j0 + 8 * k + s < n) w[k] |= (uint64_t)__ldg(piece + j0 + 8 * k + s) << (8 * s);
        }
        if (j0 + E < n) bnext = (uint32_t)__ldg(piece + j0 + E);
        auto byte_of = [&](int s) -> uint32_t {               // s is a compile-time constant after unrolling
            return s < E ? (uint32_t)(w[s >> 3] >> (8 * (s & 7))) & 0xFFu : bnext;
        };
        // ---- whole-piece probe (src/lib.rs:367-368): only a token of exactly this length can match --------------
        if (T.n_long_tokens) {
            uint64_t hsh = 0;
            if ((uint32_t)n <= T.max_token_len) {
#pragma unroll
                for (int k = 0; k < NW; k++)
                    if (j0 + 8 * k < n) hsh ^= long_hash_word(w[k], (uint32_t)(NW * gl + k));
            }
#pragma unroll
            for (int o = 1; o < G; o <<= 1) hsh ^= __shfl_xor_sync(0xFFFFFFFFu, hsh, o);
            uint32_t r = RANK_MAX;
            if (have && gl == 0 && (uint32_t)n <= T.max_token_len)
                r = piece_lookup_long(T, hsh ^ long_hash_init((uint64_t)n), (uint32_t)n, [&](uint32_t i) { return piece[i]; });
            r = __shfl_sync(0xFFFFFFFFu, r, gb);
            if (r != RANK_MAX) { if (gl == 0) { out[0] = r; long_piece_done(q, qi, 1); } n = 0; }
        }
        // ---- initial parts: one per byte (8 at a time: the table loads of a block are issued before its stores) --
        uint32_t live = 0;
#pragma unroll
        for (int hh = 0; hh < E; hh += 8) {
            uint32_t iv[8], kv[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int s = hh + k;
                iv[k] = 0; kv[k] = MIDG_NONE;
                if (j0 + s < n) {
                    iv[k] = __ldg(T.byte_id + byte_of(s));
                    if (j0 + s + 1 < n) {
                        const uint32_t r = __ldg(T.pair2 + (byte_of(s) << 8 | byte_of(s + 1)));
                        if (r != RANK_MAX) kv[k] = (r << MIDG_POS_BITS) | (uint32_t)(j0 + s);
                    }
                    live |= 1u << s;
                }
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int s = hh + k, j = j0 + s;
                idc[s * 32] = iv[k]; keyc[s * 32] = kv[k];
                linkc[s * 32] = (j + 1 < n ? (uint32_t)(j + 1) : MIDG_NIL) | ((j > 0 && j < n ? (uint32_t)(j - 1) : MIDG_NIL) << 16);
            }
        }
        __syncwarp();
        // ---- merge rounds -----------------------------------------------------------------------------------
        // A round commits the global minimum (merge 1) and, when it can be proven to be the sequential loop's NEXT step,
        // a second merge: let pair 2 be the leftmost smallest pair once merge 1 and the two pairs it invalidates are
        // taken out.  Sequentially the loop would choose between pair 2 and the two pairs merge 1 creates; if rank(pair 2)
        // is strictly below both new ranks, pair 2 is next (every other old pair is no smaller, ties leftmost) -- so both
        // merges are applied in this round, with all four neighbour probes in flight together.  Otherwise only merge 1
        // is committed and the next round starts from the exact sequential state.  (A round is bound by the latency of
        // the pair-table probes; two merges per round almost halve the number of rounds.)
        constexpr bool DUAL = G >= 4;
        auto pack = [&](uint32_t r, uint32_t pos) -> uint32_t { return r != RANK_MAX ? ((r << MIDG_POS_BITS) | pos) : MIDG_NONE; };
        auto argmin = [&]() -> uint32_t {
            uint32_t m = MIDG_NONE;
#pragma unroll
            for (int s = 0; s < E; s++) m = min(m, keyc[s * 32]);
#pragma unroll
            for (int o = 1; o < G; o <<= 1) m = min(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
            return m;
        };
        for (;;) {
            const uint32_t g1 = argmin();
            const bool act1 = g1 != MIDG_NONE;
            if (!__any_sync(0xFFFFFFFFu, act1)) break;
            const uint32_t best1 = g1 >> MIDG_POS_BITS;               // rank of the merged token == its id
            const uint32_t bj1 = act1 ? (g1 & ((1u << MIDG_POS_BITS) - 1u)) : 0u;
            // the part right of bj (it exists: key[bj] is the rank of (bj, next)), the one after it, the one before bj
            const uint32_t lka = S.link[at(bj1)];
            const uint32_t j2a = act1 ? (lka & 0xFFFFu) : 0u, jpa = lka >> 16;
            const uint32_t j3a = S.link[at(j2a)] & 0xFFFFu;
            const bool need_r1 = act1 && j3a != MIDG_NIL, need_l1 = act1 && jpa != MIDG_NIL;
            if (act1) {                                                // structure of merge 1; its two new ranks follow below
                if (gl == 0) {
                    S.id[at(bj1)] = best1;
                    S.key[at(bj1)] = MIDG_NONE; S.key[at(j2a)] = MIDG_NONE;
                    if (need_l1) S.key[at(jpa)] = MIDG_NONE;
                    S.link[at(bj1)] = j3a | (jpa << 16);
                    if (need_r1) { const uint32_t lk3 = S.link[at(j3a)]; S.link[at(j3a)] = (lk3 & 0xFFFFu) | (bj1 << 16); }
                }
                if ((uint32_t)gl == (j2a >> LOG_E)) live &= ~(1u << (j2a & (E - 1)));
            }
            __syncwarp();
            uint32_t best2 = 0, bj2 = 0, j2b = 0, jpb = MIDG_NIL, j3b = MIDG_NIL; bool act2 = false;
            if (DUAL) {
                const uint32_t g2 = argmin();                          // the pairs of merge 1 are out of the way
                act2 = act1 && g2 != MIDG_NONE;
                best2 = g2 >> MIDG_POS_BITS;
                bj2 = act2 ? (g2 & ((1u << MIDG_POS_BITS) - 1u)) : 0u;
                const uint32_t lkb = S.link[at(bj2)];                  // links already reflect merge 1
                j2b = act2 ? (lkb & 0xFFFFu) : 0u; jpb = lkb >> 16;
                j3b = S.link[at(j2b)] & 0xFFFFu;
            }
            const bool need_r2 = act2 && j3b != MIDG_NIL, need_l2 = act2 && jpb != MIDG_NIL;
            // the neighbour probes (src/lib.rs:178-194) on four lanes of the group at once
            uint32_t a = 0, b = 0; bool pr = false;
            if (gl == 0 && need_r1) { a = best1; b = S.id[at(j3a)]; pr = true; }
            if (gl == 1 && need_l1) { a = S.id[at(jpa)]; b = best1; pr = true; }
            if (DUAL && gl == 2 && need_r2) { a = best2; b = S.id[at(j3b)]; pr = true; }
            if (DUAL && gl == 3 && need_l2) { a = S.id[at(jpb)]; b = best2; pr = true; }
            uint32_t r = RANK_MAX;
            {
                uint32_t sidx = pair_start(T, a, b);
                while (__any_sync(0xFFFFFFFFu, pr))
                    if (pr) pr = !pair_step(T, pair_slot(T, sidx), a, b, sidx, r);
            }
            const uint32_t r1r = __shfl_sync(0xFFFFFFFFu, r, gb), r1l = __shfl_sync(0xFFFFFFFFu, r, gb + 1);
            uint32_t r2r = RANK_MAX, r2l = RANK_MAX;
            if (DUAL) { r2r = __shfl_sync(0xFFFFFFFFu, r, gb + 2); r2l = __shfl_sync(0xFFFFFFFFu, r, gb + 3); }
            const bool dual = act2 && best2 < r1r && best2 < r1l;      // RANK_MAX (no such pair) is above every rank
            if (act1) {
                if (gl == 0) {
                    S.key[at(bj1)] = need_r1 ? pack(r1r, bj1) : MIDG_NONE;
                    if (need_l1) S.key[at(jpa)] = pack(r1l, jpa);
                    if (dual) {                                        // merge 2, on top of merge 1 (it may consume one of its neighbours)
                        S.id[at(bj2)] = best2;
                        S.key[at(j2b)] = MIDG_NONE;
                        S.key[at(bj2)] = need_r2 ? pack(r2r, bj2) : MIDG_NONE;
                        if (need_l2) S.key[at(jpb)] = pack(r2l, jpb);
                        S.link[at(bj2)] = j3b | (jpb << 16);
                        if (need_r2) { const uint32_t lk3 = S.link[at(j3b)]; S.link[at(j3b)] = (lk3 & 0xFFFFu) | (bj2 << 16); }
                    }
                }
                if (dual && (uint32_t)gl == (j2b >> LOG_E)) live &= ~(1u << (j2b & (E - 1)));
            }
            __syncwarp();
        }
        // ---- tokens: the live parts, left to right ------------------------------------------------------------
        {
            const uint32_t c = (uint32_t)__popc(live);
            uint32_t inc = c;
#pragma unroll
            for (int o = 1; o < G; o <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (gl >= o) inc += y; }
            const uint32_t total = __shfl_sync(0xFFFFFFFFu, inc, gb + G - 1);
            uint32_t o = inc - c; bool bad = false;
            for (uint32_t m = live; m;) {
                const int s = __ffs((int)m) - 1; m &= m - 1;
                const uint32_t x = idc[s * 32];
                out[o++] = x; bad |= x >= PSEUDO_BASE;
            }
            if (bad) atomicOr(&ctr->err, ERR_NOBYTE);
            if (have && n && gl == 0) long_piece_done(q, qi, total);
        }
        __syncwarp();
    }
}

// 32 parts per lane (12 KiB of state per warp): 257..1024, 129..256 and 65..128 bytes
__global__ void __launch_bounds__(MIDG_WARPS * 32, 4) mid_group32_kernel(const uint8_t *__restrict__ text, DevTables T, LongQ q,
                                                                        uint32_t *ltok, Counters *ctr, int max_cls) {
    __shared__ MidGSmem<32> smem[MIDG_WARPS];
    MidGSmem<32> &S = smem[threadIdx.x >> 5];
    if (max_cls >= 4) midg_class<32, 32>(text, T, q, 4, ltok, ctr, S);
    if (max_cls >= 3) midg_class<8, 32>(text, T, q, 3, ltok, ctr, S);
    midg_class<4, 32>(text, T, q, 2, ltok, ctr, S);
}

// 16 parts per lane (6 KiB of state per warp): 33..64 and 17..32 bytes
__global__ void __launch_bounds__(MIDG_WARPS * 32, 9) mid_group16_kernel(const uint8_t *__restrict__ text, DevTables T, LongQ q,
                                                                        uint32_t *ltok, Counters *ctr, int max_cls) {
    __shared__ MidGSmem<16> smem[MIDG_WARPS];
    MidGSmem<16> &S = smem[threadIdx.x >> 5];
    if (max_cls >= 1) midg_class<4, 16>(text, T, q, 1, ltok, ctr, S);
    midg_class<2, 16>(text, T, q, 0, ltok, ctr, S);
}
