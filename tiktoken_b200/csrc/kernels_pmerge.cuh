// kernels_pmerge.cuh -- pieces of 17..256 bytes (CJK runs, indentation, separators, long identifiers): the SEGMENTED
// PARALLEL MERGE.  A warp takes a batch of pieces of one length class (one piece of <= 256 or <= 1024 bytes as shipped;
// the code packs several shorter ones) into a buffer of parts in shared memory and merges them together, a handful of
// ROUNDS for the whole batch instead of one round per merge and piece.
//
// `_byte_pair_merge` (src/lib.rs:140-196) merges ONE pair per step: the smallest rank, leftmost on ties.  If merges
// never created pairs, that loop would walk the pairs in (rank, position) order and take a pair unless a neighbour was
// taken before it -- the greedy independent set of the path in key order.  It has a closed form: pair e is taken iff
// the run of increasing keys that ends at e coming from the left and the one coming from the right both have even
// length (valleys are taken, then every second pair up a slope, a peak only if both slopes agree); the parities of all
// runs of a batch come out of two carry-propagating additions on the "key(e-1) < key(e)" bitmap (the trick that finds
// odd-length backslash runs in SIMD JSON parsers), across words with a ballot carry-lookahead.
// The pairs that merges DO create are the only thing that can disturb that order.  So a round
//   1. takes the independent set G,
//   2. probes, for every member, the ranks of the two pairs its merge creates (its neighbour being the merged token
//      when the pair two places away is in G with a smaller key, else the part as it stands) -- all probes of a round in flight together,
//   3. commits the members whose rank is strictly below T = the smallest rank any member of its piece would create (a
//      prefix of the sequential order in which no new pair can have come first), plus, always, the piece's global
//      minimum (the sequential loop's next step whatever it creates),
// and the next round starts from that exact sequential state.  Exact on arbitrary (adversarial, non-monotone)
// vocabularies: tests/test_parallel_merge_model.py states the round as an executable model against the sequential loop, the
// GPU parity tests check this kernel.  Measured on the mixed-script corpus: 4-6 rounds per piece where the sequential loop
// takes 30-120 merges.  Pieces are segments of the buffer: the last part of a piece carries the separator rank PM_SEP
// ("no pair across pieces"), so nothing ever looks across a piece boundary.
// Keys pack (rank << 10 | position) for the per-piece minimum: vocabularies with ranks of 2^22 and above keep the
// lane-per-piece kernels of kernels_long.cuh.
#pragma once
#include "dev_common.cuh"

using namespace b2bpe;

static const int PM_WARPS = 4;                    // warps per block (independent of each other)
static const int PM_MAXSEG = 16;                  // pieces per batch (17..32-byte class)
static const uint32_t PM_SEP = 0xFFFFFFFEu;       // rank slot of the LAST part of a piece; RANK_MAX: no such pair in the vocabulary
static const int PM_POS_BITS = 10;

template <int PM_CAP>
struct PMergeSmem {                               // 9.7 KiB per warp with 512 parts
    static const int PM_WORDS = PM_CAP / 32;
    uint32_t id[PM_CAP];                          // token id of the part
    uint32_t rk[PM_CAP + 2];                      // rank of (this part, next part); PM_SEP on the last part of a piece
    uint32_t nl[PM_CAP], nr[PM_CAP];              // ranks of the two pairs the merge at e creates
    uint16_t list[PM_CAP];                        // the members of the independent set, dense (the probes run with all lanes busy)
    uint8_t seg[PM_CAP];                          // piece index within the batch
    uint32_t tbits[PM_WORDS + 2], cbits[PM_WORDS + 2];   // taken / committed bitmaps, one zero word of padding on either side
    uint32_t T[PM_MAXSEG], c1[PM_MAXSEG];         // per piece: smallest created rank; smallest (rank << 10 | position)
    uint32_t seg_lo[PM_MAXSEG], seg_hi[PM_MAXSEG];
    unsigned long long pst[PM_MAXSEG];            // byte offset of piece s
};

// Bit e of the result is set iff bit e of `w` is set and its distance to the START of its run of ones is even.  Lane t
// holds word t of a 1024-bit map.  Runs that start at an even position are cleared by adding 1 at their start (the carry
// ripples through the run and across words); the others are what is left.
__device__ __forceinline__ uint32_t pm_alt_from_start(uint32_t w, int lane) {
    const uint32_t prev = __shfl_up_sync(0xFFFFFFFFu, w, 1);
    const uint32_t prev_msb = lane ? prev >> 31 : 0u;
    const uint32_t starts = w & ~((w << 1) | prev_msb);
    uint32_t s = w + (starts & 0x55555555u);
    const uint32_t G = __ballot_sync(0xFFFFFFFFu, s < w);                 // carry out
    const uint32_t P = __ballot_sync(0xFFFFFFFFu, s == 0xFFFFFFFFu);      // would pass a carry on
    const uint32_t cin = ((G | P) + G) ^ (P & ~G);                        // bit t: carry INTO word t  (carry-lookahead as an addition)
    s += (cin >> lane) & 1u;
    const uint32_t even_runs = w & ~s;
    return (even_runs & 0x55555555u) | (w & ~even_runs & 0xAAAAAAAAu);
}
// the same, distance to the END of the run: mirror the map (1024 bits: position parity flips consistently)
__device__ __forceinline__ uint32_t pm_alt_from_end(uint32_t w, int lane) {
    const uint32_t r = __shfl_sync(0xFFFFFFFFu, __brev(w), 31 - lane);
    const uint32_t x = pm_alt_from_start(r, lane);
    return __shfl_sync(0xFFFFFFFFu, __brev(x), 31 - lane);
}

// SINGLE: one piece per batch (as shipped) -- no piece-index array, and the per-piece minima of a round come out of a warp
// reduction instead of shared-memory atomics (the kernel is bound by shared-memory wavefronts).
template <int PM_CAP, bool SINGLE>
__device__ void pmerge_class(const uint8_t *__restrict__ text, const DevTables &T, const LongQ &q, int cls, int per_batch,
                             uint32_t *ltok, Counters *ctr, PMergeSmem<PM_CAP> &S) {
    const int lane = threadIdx.x & 31;
    const uint32_t lt_mask = (1u << lane) - 1u;
    const unsigned int n_items = ctr->n_cls[cls];
    const unsigned int *list = q.cls[cls];
    for (;;) {
        unsigned int k0 = 0;
        if (lane == 0) k0 = atomicAdd(&ctr->cls_head[cls], (unsigned int)per_batch);
        k0 = __shfl_sync(0xFFFFFFFFu, k0, 0);
        if (k0 >= n_items) break;
        const int np = (int)min((unsigned int)per_batch, n_items - k0);
        // ---- the batch: lane s describes piece s ------------------------------------------------------------
        unsigned int qi = 0; unsigned long long st = 0; uint32_t n = 0;
        if (lane < np) { qi = list[k0 + lane]; st = q.start[qi]; n = q.len[qi]; }
        // whole-piece probe (src/lib.rs:367-368): only a token of exactly this length can match
        if (T.n_long_tokens) {
            for (int s = 0; s < np; s++) {
                const uint32_t ns = __shfl_sync(0xFFFFFFFFu, n, s);
                if (ns > T.max_token_len) continue;
                const uint8_t *piece = text + __shfl_sync(0xFFFFFFFFu, st, s);
                uint64_t hsh = 0;
                for (uint32_t k = lane; 8 * k < ns; k += 32) {
                    uint64_t w = 0;
                    for (uint32_t b = 0; b < 8 && 8 * k + b < ns; b++) w |= (uint64_t)__ldg(piece + 8 * k + b) << (8 * b);
                    hsh ^= long_hash_word(w, k);
                }
#pragma unroll
                for (int o = 16; o; o >>= 1) hsh ^= __shfl_xor_sync(0xFFFFFFFFu, hsh, o);
                uint32_t r = RANK_MAX;
                if (lane == 0) r = piece_lookup_long(T, hsh ^ long_hash_init((uint64_t)ns), ns, [&](uint32_t i) { return piece[i]; });
                r = __shfl_sync(0xFFFFFFFFu, r, 0);
                if (r != RANK_MAX && lane == s) { ltok[st] = r; long_piece_done(q, qi, 1); n = 0; }
            }
        }
        const uint32_t ninc = warp_incl_scan_u32(n, lane);
        uint32_t m = __shfl_sync(0xFFFFFFFFu, ninc, 31);                  // parts in the buffer (<= PM_CAP by the class limits)
        const uint32_t base = ninc - n;
        for (int s = 0; s < np; s++) {                                    // one part per byte
            const uint32_t ns = __shfl_sync(0xFFFFFFFFu, n, s), bs = __shfl_sync(0xFFFFFFFFu, base, s);
            const uint8_t *piece = text + __shfl_sync(0xFFFFFFFFu, st, s);
            for (uint32_t j = lane; j < ns; j += 32) {
                const uint32_t b = __ldg(piece + j);
                S.id[bs + j] = __ldg(T.byte_id + b);
                S.rk[bs + j] = j + 1 < ns ? __ldg(T.pair2 + (b << 8 | __ldg(piece + j + 1))) : PM_SEP;
                if (!SINGLE) S.seg[bs + j] = (uint8_t)s;
            }
        }
        if (lane < 2) S.rk[m + lane] = RANK_MAX;
        if (lane == 0) { S.tbits[0] = 0; S.cbits[0] = 0; }
        if (lane < np) S.pst[lane] = st;
        __syncwarp();
        uint32_t *const id = S.id, *const rk = S.rk; uint8_t *const seg = S.seg;
        // ---- rounds --------------------------------------------------------------------------------------------
        for (int round = 0; m; round++) {
            if (round > PM_CAP) { if (lane == 0) atomicOr(&ctr->err, ERR_INTERNAL); break; }   // every round merges: cannot happen
            const int nw = (int)((m + 31) >> 5);
            // 1. bitmaps: U(e) = key(e-1) < key(e) in (rank, position) order (ones beyond the end), V(e) = mergeable
            uint32_t myU = 0xFFFFFFFFu, myV = 0, carry = RANK_MAX;       // carry: the rank slot before this iteration's first part
            for (int t = 0; t < nw; t++) {
                const uint32_t e = 32u * t + lane;
                const uint32_t r0 = e < m ? rk[e] : RANK_MAX;
                const uint32_t up = __shfl_up_sync(0xFFFFFFFFu, r0, 1);    // the left neighbour's slot from its lane, not from shared memory
                const uint32_t rm1 = lane ? up : carry;
                carry = __shfl_sync(0xFFFFFFFFu, r0, 31);
                const uint32_t ub = __ballot_sync(0xFFFFFFFFu, e >= m || (e >= 1 && rm1 <= r0));
                const uint32_t vb = __ballot_sync(0xFFFFFFFFu, r0 < PM_SEP);
                if (lane == t) { myU = ub; myV = vb; }
            }
            if (!__any_sync(0xFFFFFFFFu, myV != 0)) break;               // nothing left to merge in any piece
            // 2. the independent set: both run lengths even; its members as a dense list
            uint32_t n_taken;
            {
                const uint32_t odd_l = pm_alt_from_start(myU, lane);      // odd number of increasing steps end at e from the left
                const uint32_t nextU = __shfl_down_sync(0xFFFFFFFFu, myU, 1);
                const uint32_t zs = ~__funnelshift_r(myU, lane == 31 ? 0xFFFFFFFFu : nextU, 1);   // Z'(e) = key(e+1) < key(e)
                const uint32_t odd_r = pm_alt_from_end(zs, lane);
                const uint32_t tk = lane < nw ? (myV & ~odd_l & ~odd_r) : 0u;
                if (lane < nw) S.tbits[1 + lane] = tk;
                if (lane == 0) S.tbits[1 + nw] = 0;
                if (lane < np) { S.T[lane] = RANK_MAX; S.c1[lane] = RANK_MAX; }
                const uint32_t c = __popc(tk), inc = warp_incl_scan_u32(c, lane);
                n_taken = __shfl_sync(0xFFFFFFFFu, inc, 31);
                // a list entry = position (10 bits) | "the pair two places to the left / right is a member too" (bits 10, 11):
                // the probes then need no look-ups in the bitmap
                const uint32_t prevw = __shfl_up_sync(0xFFFFFFFFu, tk, 1), nextw = __shfl_down_sync(0xFFFFFFFFu, tk, 1);
                const uint32_t tm2 = (tk << 2) | (lane ? prevw >> 30 : 0u), tp2 = (tk >> 2) | (lane < 31 ? nextw << 30 : 0u);
                uint16_t *dst = S.list + (inc - c);
                for (uint32_t mm = tk; mm; mm &= mm - 1) {
                    const int j = __ffs(mm) - 1;
                    *dst++ = (uint16_t)((32 * lane + j) | (((tm2 >> j) & 1u) << 10) | (((tp2 >> j) & 1u) << 11));
                }
            }
            __syncwarp();
            // 3. the two pairs every member's merge creates -- all lanes busy, four table loads in flight per lane
            uint32_t myT = RANK_MAX, myC1 = RANK_MAX;
            for (uint32_t i = lane; i < n_taken; i += 32) {
                const uint32_t ent = S.list[i], e = ent & 1023u;
                const uint32_t r0 = rk[e];
                const bool has_l = e >= 1 && rk[e - 1] != PM_SEP;        // a part of the same piece to the left
                const bool has_r = rk[e + 1] != PM_SEP;                  // ... after the pair, to the right
                uint32_t L = 0, R = 0;
                if (has_l) {
                    const uint32_t r2 = e >= 2 ? rk[e - 2] : RANK_MAX;
                    L = ((ent >> 10) & 1u) && r2 <= r0 ? r2 : id[e - 1];
                }
                if (has_r) {
                    const uint32_t r2 = rk[e + 2];
                    R = ((ent >> 11) & 1u) && r2 < r0 ? r2 : id[e + 2];
                }
                uint32_t vl = RANK_MAX, vr = RANK_MAX;
                if (has_l && has_r) pair_lookup2(T, L, r0, r0, R, vl, vr);
                else if (has_l) vl = pair_lookup(T, L, r0);
                else if (has_r) vr = pair_lookup(T, r0, R);
                S.nl[e] = vl; S.nr[e] = has_r ? vr : PM_SEP;             // no right part: the merged part becomes the last one of its piece
                if (SINGLE) { myT = min(myT, min(vl, vr)); myC1 = min(myC1, (r0 << PM_POS_BITS) | e); }
                else {
                    const uint32_t s = seg[e];
                    atomicMin(&S.T[s], min(vl, vr));
                    atomicMin(&S.c1[s], (r0 << PM_POS_BITS) | e);
                }
            }
            if (SINGLE) { myT = warp_min_u32(myT); myC1 = warp_min_u32(myC1) & ((1u << PM_POS_BITS) - 1u); }
            __syncwarp();
            // 4a. commit: below every created rank of the piece, or the piece's minimum
            for (int t = 0; t < nw; t++) {
                const uint32_t e = 32u * t + lane;
                bool com = (S.tbits[1 + t] >> lane) & 1u;
                if (com) {
                    if (SINGLE) com = rk[e] < myT || e == myC1;
                    else { const uint32_t s = seg[e]; com = rk[e] < S.T[s] || e == (S.c1[s] & ((1u << PM_POS_BITS) - 1u)); }
                }
                const uint32_t cb = __ballot_sync(0xFFFFFFFFu, com);
                if (lane == 0) S.cbits[1 + t] = cb;
            }
            if (lane == 0) S.cbits[1 + nw] = 0;
            __syncwarp();
            // 4b. compaction in place: merged parts, their new ranks, absorbed parts dropped.  Iteration t only reads parts
            //     >= 32 t and only writes positions <= 32 t + 31, after all its reads.
            uint32_t out = 0;
            for (int t = 0; t < nw; t++) {
                const uint32_t e = 32u * t + lane;
                const uint32_t cw = S.cbits[1 + t], cprev = S.cbits[t], cnext = S.cbits[2 + t];
                const bool com_e = (cw >> lane) & 1u;
                const bool com_m1 = (((cw << 1) | (cprev >> 31)) >> lane) & 1u;
                const bool com_p1 = (((cw >> 1) | (cnext << 31)) >> lane) & 1u;
                const bool com_p2 = (((cw >> 2) | (cnext << 30)) >> lane) & 1u;
                const bool keep = e < m && !com_m1;
                uint32_t nid = 0, nrk = 0, sg = 0;
                if (keep) {
                    const uint32_t r0 = rk[e];
                    if (!SINGLE) sg = seg[e];
                    if (com_e) {                                     // (the pair two places on only counts inside the same piece)
                        nid = r0; nrk = S.nr[e];
                        if (nrk != PM_SEP && com_p2 && r0 <= rk[e + 2]) nrk = S.nl[e + 2];
                    } else { nid = id[e]; nrk = r0 == PM_SEP ? PM_SEP : (com_p1 ? S.nl[e + 1] : r0); }
                }
                const uint32_t kb = __ballot_sync(0xFFFFFFFFu, keep);
                __syncwarp();
                if (keep) {
                    const uint32_t pos = out + __popc(kb & lt_mask);
                    id[pos] = nid; rk[pos] = nrk; if (!SINGLE) seg[pos] = (uint8_t)sg;
                }
                out += __popc(kb);
                __syncwarp();
            }
            m = out;
            if (lane < 2) rk[m + lane] = RANK_MAX;
            __syncwarp();
        }
        // ---- tokens: the parts of every piece, left to right ----------------------------------------------------------
        {
            if (SINGLE) { if (lane == 0) { S.seg_lo[0] = 0; S.seg_hi[0] = m; } }
            else for (uint32_t e = lane; e < m; e += 32) {
                const uint32_t s = seg[e];
                if (e == 0 || seg[e - 1] != s) S.seg_lo[s] = e;
                if (e + 1 == m || seg[e + 1] != s) S.seg_hi[s] = e + 1;
            }
            __syncwarp();
            bool bad = false;
            for (uint32_t e = lane; e < m; e += 32) {
                const uint32_t s = SINGLE ? 0u : (uint32_t)seg[e];
                const uint32_t x = id[e];
                ltok[S.pst[s] + (e - S.seg_lo[s])] = x; bad |= x >= PSEUDO_BASE;
            }
            if (bad) atomicOr(&ctr->err, ERR_NOBYTE);
            if (lane < np && n) long_piece_done(q, qi, S.seg_hi[lane] - S.seg_lo[lane]);
        }
        __syncwarp();
    }
}

// One piece per buffer of CAP parts, CAP = the upper length of the class: 129..256 bytes -> 256 parts (4.9 KiB of shared
// memory per warp, 40 warps per SM), 65..128 -> 128, 33..64 -> 64.  One piece per 256-part buffer rather than two per
// 512-part buffer (9.7 KiB, 20 warps per SM): the kernel is meant to hide latency and L1TEX waits with more warps, and
// instruction issue is not what it spends.
template <int CAP, int CLS>
__global__ void __launch_bounds__(PM_WARPS * 32) pmerge_kernel(const uint8_t *__restrict__ text, DevTables T, LongQ q, uint32_t *ltok,
                                                              Counters *ctr) {
    __shared__ PMergeSmem<CAP> smem[PM_WARPS];
    pmerge_class<CAP, true>(text, T, q, CLS, 1, ltok, ctr, smem[threadIdx.x >> 5]);
}

// 257..1024 bytes: one piece per 1024-part batch
static const int PM_WARPS_L = 2;
__global__ void __launch_bounds__(PM_WARPS_L * 32) pmerge_long_kernel(const uint8_t *__restrict__ text, DevTables T, LongQ q,
                                                                     uint32_t *ltok, Counters *ctr) {
    __shared__ PMergeSmem<1024> smem[PM_WARPS_L];
    PMergeSmem<1024> &S = smem[threadIdx.x >> 5];
    pmerge_class<1024, true>(text, T, q, CLS_G1024, 1, ltok, ctr, S);
}
