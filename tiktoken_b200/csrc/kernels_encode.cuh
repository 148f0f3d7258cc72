// kernels_encode.cuh -- encode = probe -> merge the misses -> (scan) -> gather.
//
// probe_kernel   persistent warps, one 1 KiB sub-tile at a time: the TMA unit stages the next sub-tile's text and
//                piece-start words into shared memory (cp.async.bulk + mbarrier, double buffered) while the warp works
//                on the current one; the piece starts are compacted into a list (all 32 lanes busy whatever the
//                distribution) and every piece of <= 16 bytes is probed in the piece tables (src/lib.rs:367-368), two
//                probes in flight per lane: one 16-byte load per step for a piece of <= 11 bytes, two above.  One 32-bit slot per PIECE goes to `ptok` (token id, or a tagged reference
//                to the miss queue / the long-piece queue); a miss is appended to a global queue TOGETHER WITH ITS 16
//                KEY BYTES, so that nothing downstream goes back to the text.
// miss_*         one owner per distinct missed piece (miss_dedup: a per-call memo), counting sort of the owners by
//                piece length, carrying the records; miss_kernel: one piece per lane, 32 per warp, all lanes walking
//                one convergent instruction stream (merge_short_conv), the literal min-rank loop of _byte_pair_merge
//                (src/lib.rs:140-196), reading dense sorted records; miss_fanout: every other occurrence copies its
//                owner's result.
// gather_kernel  one warp per sub-tile, PIECE-parallel: 32 slots per step -> token counts -> warp scan -> tokens and
//                per-document offsets written at their final position.
// Kernel boundaries do the ordering; there is no look-back chain and no ticket counter.
#pragma once
#include "dev_common.cuh"

using namespace b2bpe;

static const uint32_t PT_MISS = 0x40000000u, PT_LONG = 0x80000000u, PT_KIND = 0xC0000000u, PT_PAYLOAD = 0x3FFFFFFFu;
static const uint32_t PT_EMPTY = 0xFFFFFFFFu;             // zero-token slot (only on error / retry paths)

struct MissQ {                // queue of pieces (2..16 bytes) that are not tokens themselves
    uint4 *key;               // the piece bytes, little-endian words, zero padded            (queue order)
    uint32_t *pos;            // byte offset of the piece
    uint32_t *roff;           // offset of its result region in mres (sum of lengths => tokens always fit)
    uint8_t *len;
    uint4 *rec;               // result record (written by miss_kernel): {tokens produced, first three tokens}; the rest, if any, in mres
    uint4 *skey;              // keys sorted by piece length (so that a warp merges pieces of one length)
    uint4 *smeta;             // {queue index, roff, pos, len} in the same order
    uint32_t cap;             // capacity of the queue (entries)
    unsigned long long mres_cap;   // capacity of mres (tokens)
};

// Miss memo of one call: the first occurrence of each distinct missed piece becomes its owner and is the only one merged;
// the other occurrences copy the owner's result.  Cleared by every call, so a result never depends on an earlier one.
struct MissMemo {
    uint4 *key;               // [mask + 1] memo_key of the piece in the slot, 0: empty
    uint32_t *owner;          // [mask + 1] queue index of the slot's owner
    uint32_t *slot;           // [queue] memo slot of a duplicate (written for duplicates only)
    uint32_t *own;            // [queue] per dedup block, in its range of the queue: owners from the front, duplicates from the back
    uint32_t *block_n;        // [dedup blocks][2] owners and duplicates found by the block
    uint32_t mask;            // slots - 1 (slots: a power of two)
    uint32_t limit;           // slots a dedup block may take: half of them, shared out equally
    uint32_t on;              // 0: every missed piece is its own owner
};
static const int MEMO_PROBES = 8;                        // linear probe steps before a piece gives up and owns itself
static const uint32_t MEMO_TRIAL = 256;                  // slots a dedup block takes before it checks that the memo pays

struct TileParams {
    const uint8_t *text; long long n_bytes; long long n_words; long long n_sub;
    const uint32_t *pbits; const uint32_t *dbits; const uint32_t *span_first_doc;
    const unsigned long long *doc_off; unsigned long long n_docs;
    LongQ q; const uint32_t *lidx; const uint32_t *ltok;
    const uint32_t *doc_tiles;    // sub-tiles with a document start (sparse-document batches), count in ctr->n_doc_tiles
    const uint32_t *sbits;        // special-piece mask (NULL unless the call handles special tokens): id at ltok[start]
    uint32_t *ptok;               // [n_sub][SUB_BYTES] one slot per piece, in piece order
    MissQ mq; uint32_t *mres;     // miss queue and its token results
    uint32_t *sub_count;          // [n_sub] tokens emitted by the sub-tile
    unsigned long long *sub_base; // [n_sub+1] exclusive prefix of sub_count
    uint32_t *out; unsigned long long *tok_off;
    unsigned long long *big_dst, *big_src; uint32_t *big_n;   // token copies too large for one warp (big_copy_kernel)
    Counters *ctr;
};

static const int ENC_WARPS = 4;                          // warps per block
// probe_kernel grid: 12 blocks per SM where 10 fit at once, so a block's share of the strided sub-tiles is smaller and
// blocks that do not fit yet start as others finish.  Measured on an H100 80GB HBM3 at 700 W, config 2: probe_kernel
// 3.2 ms with 10, 3.0 with 12, 3.4 with 16 (DESIGN §9)
static const int PROBE_BLOCKS_PER_SM = 12;
static const int SUB_BYTES = 1024;                       // bytes per warp sub-tile (also: max pieces per sub-tile)
static const int STAGE_TEXT = SUB_BYTES + 32;            // staged text: the sub-tile + 32 bytes of look-ahead
static const int STAGE_PW = 36;                          // staged piece-start words: 32 own + 2 look-ahead (+2: 16-byte multiple)

struct ProbeSmem {
    __align__(16) uint8_t text[2][STAGE_TEXT];
    __align__(16) uint32_t p[2][STAGE_PW];
    __align__(8) unsigned long long mbar[2];
    uint32_t nmiss;
    uint16_t plist[SUB_BYTES + 2];     // piece start offsets of the sub-tile, in order, + end sentinel
    uint16_t miss[SUB_BYTES / 2];      // piece indices (into plist) of the misses
};

// the <= 16 bytes of a piece at an arbitrary offset of the staged text: five aligned words + funnel shifts, masked to len
__device__ __forceinline__ void load_key(const uint8_t *txt, int off, int len, uint32_t &a0, uint32_t &a1, uint32_t &a2, uint32_t &a3) {
    const uint32_t *wp = reinterpret_cast<const uint32_t *>(txt) + (off >> 2);
    const int sh = (off & 3) * 8;
    const uint32_t w0 = wp[0], w1 = wp[1], w2 = wp[2], w3 = wp[3], w4 = wp[4];
    const int nb = len * 8;
    a0 = __funnelshift_r(w0, w1, sh) & low_mask_clamped(nb);
    a1 = __funnelshift_r(w1, w2, sh) & low_mask_clamped(nb - 32);
    a2 = __funnelshift_r(w2, w3, sh) & low_mask_clamped(nb - 64);
    a3 = __funnelshift_r(w3, w4, sh) & low_mask_clamped(nb - 96);
}

__global__ void __launch_bounds__(ENC_WARPS * 32) probe_kernel(TileParams p, DevTables T) {
    __shared__ ProbeSmem smem[ENC_WARPS];
    ProbeSmem &S = smem[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * ENC_WARPS;
    long long sub = (long long)blockIdx.x * ENC_WARPS + (threadIdx.x >> 5);
    if (sub >= p.n_sub) return;                          // warps are independent: no block barrier below
    // shared-memory addresses of buffer b are base + b * size: computed, not taken from an array indexed by the run-time
    // buffer number (such an array lives in local memory)
    const uint32_t mb0 = smem_u32(&S.mbar[0]), s_text0 = smem_u32(S.text[0]), s_pw0 = smem_u32(S.p[0]);
    auto mb = [&](int b) -> uint32_t { return mb0 + (uint32_t)b * (uint32_t)sizeof(S.mbar[0]); };
    const uint64_t pol = l2_policy_evict_first();        // the text is streamed once: do not let it displace the tables in L2
    if (lane == 0) { mbar_init(mb(0), 1); mbar_init(mb(1), 1); mbar_fence_init(); }
    __syncwarp();
    // TMA staging of sub-tile t into buffer b (lane 0): text (readable up to n_bytes + 16) and piece-start words
    auto stage = [&](long long t, int b) {
        const long long left = p.n_bytes - t * SUB_BYTES;
        const uint32_t tbytes = left >= STAGE_TEXT ? (uint32_t)STAGE_TEXT : (uint32_t)((left + 15) & ~15ll);
        mbar_arrive_expect_tx(mb(b), tbytes + STAGE_PW * 4);
        if (tbytes) tma_load_1d(s_text0 + (uint32_t)b * (uint32_t)sizeof(S.text[0]), p.text + t * SUB_BYTES, tbytes, mb(b), pol);
        tma_load_1d(s_pw0 + (uint32_t)b * (uint32_t)sizeof(S.p[0]), p.pbits + t * 32, STAGE_PW * 4, mb(b), pol);
    };
    if (lane == 0) stage(sub, 0);
    int cur = 0; uint32_t phase = 0;                      // bit b of `phase` = parity to wait for on buffer b
    for (; sub < p.n_sub; sub += stride, cur ^= 1) {
        if (lane == 0 && sub + stride < p.n_sub) stage(sub + stride, cur ^ 1);   // overlaps with this sub-tile's probes
        mbar_wait(mb(cur), (phase >> cur) & 1u);
        phase ^= 1u << cur;
        const uint8_t *txt = S.text[cur];
        const uint32_t *pw = S.p[cur];
        const long long sub_byte = sub * SUB_BYTES;
        uint32_t *const slot = p.ptok + sub * SUB_BYTES;
        if (lane == 0) S.nmiss = 0;

        // ---- piece list ------------------------------------------------------------------------
        uint32_t pv = pw[lane];
        {
            const long long span0 = sub_byte + lane * 32;
            if (span0 + 32 > p.n_bytes) {                      // drop the end sentinel / bits beyond the text
                const long long keep = p.n_bytes - span0;
                pv = keep <= 0 ? 0u : (pv & ((1u << keep) - 1u));
            }
        }
        uint32_t np;
        {
            const uint32_t c = __popc(pv);
            const uint32_t inc = warp_incl_scan_u32(c, lane);
            np = __shfl_sync(0xFFFFFFFFu, inc, 31);
            uint16_t *dst = S.plist + (inc - c);
            for (uint32_t m = pv; m;) { const int j = __ffs(m) - 1; m &= m - 1; *dst++ = (uint16_t)(lane * 32 + j); }
            if (lane == 0) {                                   // end sentinel: next piece start (or "far away")
                const uint32_t nx = pw[32];
                const long long tail = p.n_bytes - sub_byte;           // text ends inside this sub-tile?
                S.plist[np] = (uint16_t)(tail <= SUB_BYTES ? tail : (nx ? SUB_BYTES + __ffs(nx) - 1 : SUB_BYTES + 32));
            }
        }
        __syncwarp();

        // ---- whole-piece probe, two pieces per lane per iteration --------------------------------
        uint32_t cnt = 0;                                      // tokens known so far (hits, single bytes)
        auto prep = [&](uint32_t i, int &len, uint32_t &a0, uint32_t &a1, uint32_t &a2, uint32_t &a3) -> int {
            if (i >= np) return 0;
            const int off = S.plist[i];
            len = (int)S.plist[i + 1] - off;
            if (p.sbits) {                                     // an allowed special token (lib.rs:426-436): its id was resolved by the scan
                const long long pos = sub_byte + off;
                if ((p.sbits[pos >> 5] >> (pos & 31)) & 1u) { st_stream_u32(slot + i, p.ltok[pos]); cnt++; return 0; }
            }
            if (len > SHORT_MAX) {                             // long path: merged by the long-piece kernels, concurrently, on a side
                const uint32_t qi = p.lidx[(sub_byte + off) >> 4];     // stream (they credit their tokens to sub_count themselves)
                st_stream_u32(slot + i, PT_LONG | qi);
                return 0;
            }
            // single-byte pieces (18 % of English) take the same path as the others: every single-byte token is in the
            // piece table, and a byte the vocabulary lacks falls out as a miss whose merge reports ERR_NOBYTE -- one
            // instruction stream for all lanes instead of a divergent branch
            load_key(txt, off, len, a0, a1, a2, a3);
            return 1;
        };
        auto finish = [&](uint32_t i, int len, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t s, U4 e0, U4 e1) {
            const uint32_t r = piece_finish(T, a0, a1, a2, a3, (uint32_t)len, s, e0, e1);   // continues from the prefetched slot
            if (r != RANK_MAX) { st_stream_u32(slot + i, r); cnt++; }
            else S.miss[atomicAdd(&S.nmiss, 1u)] = (uint16_t)i;
        };
        for (uint32_t i = lane; i < np; i += 64) {
            int lenA = 0, lenB = 0;
            uint32_t a0 = 0, a1 = 0, a2 = 0, a3 = 0, b0 = 0, b1 = 0, b2 = 0, b3 = 0;
            const int needA = prep(i, lenA, a0, a1, a2, a3);
            const int needB = prep(i + 32, lenB, b0, b1, b2, b3);
            uint32_t sA = 0, sB = 0;
            U4 eA0 = {0, 0, 0, 0}, eA1 = {0, 0, 0, 0}, eB0 = {0, 0, 0, 0}, eB1 = {0, 0, 0, 0};
            if (needA) sA = piece_issue(T, a0, a1, a2, a3, (uint32_t)lenA, eA0, eA1);
            if (needB) sB = piece_issue(T, b0, b1, b2, b3, (uint32_t)lenB, eB0, eB1);
            if (needA) finish(i, lenA, a0, a1, a2, a3, sA, eA0, eA1);
            if (needB) finish(i + 32, lenB, b0, b1, b2, b3, sB, eB0, eB1);
        }
        __syncwarp();

        // ---- misses -> global queue (one atomic per sub-tile), result space = sum of their lengths ----
        const uint32_t nmiss = S.nmiss;
        if (nmiss) {
            uint32_t run = 0;
            for (uint32_t k0 = 0; k0 < nmiss; k0 += 32) {      // total length first
                const uint32_t k = k0 + lane;
                uint32_t len = 0;
                if (k < nmiss) { const uint32_t i = S.miss[k]; len = (uint32_t)S.plist[i + 1] - S.plist[i]; }
                run += warp_sum_u32(len);
            }
            uint32_t qbase = 0; unsigned long long rbase = 0;
            if (lane == 0) {
                qbase = atomicAdd(&p.ctr->n_miss, nmiss);
                rbase = atomicAdd(&p.ctr->miss_bytes, (unsigned long long)run);
            }
            qbase = __shfl_sync(0xFFFFFFFFu, qbase, 0); rbase = __shfl_sync(0xFFFFFFFFu, rbase, 0);
            // the queue is sized from experience, not for the worst case: on overflow the counters keep counting and
            // the host re-runs the batch with the exact size (ERR_MISSCAP)
            const bool fits = (unsigned long long)qbase + nmiss <= p.mq.cap && rbase + run <= p.mq.mres_cap;
            if (!fits && lane == 0) atomicOr(&p.ctr->err, ERR_MISSCAP);
            run = 0;
            for (uint32_t k0 = 0; k0 < nmiss; k0 += 32) {
                const uint32_t k = k0 + lane;
                uint32_t i = 0, off = 0, len = 0;
                if (k < nmiss) { i = S.miss[k]; off = S.plist[i]; len = (uint32_t)S.plist[i + 1] - off; }
                const uint32_t inc = warp_incl_scan_u32(len, lane);
                if (k < nmiss) {
                    if (fits) {
                        const uint32_t qi = qbase + k;
                        uint32_t a0, a1, a2, a3;
                        load_key(txt, (int)off, (int)len, a0, a1, a2, a3);
                        st_stream_u4(p.mq.key + qi, make_uint4(a0, a1, a2, a3));
                        p.mq.pos[qi] = (uint32_t)(sub_byte + off); p.mq.len[qi] = (uint8_t)len;
                        p.mq.roff[qi] = (uint32_t)rbase + run + inc - len;
                        st_stream_u32(slot + i, PT_MISS | qi);
                    } else st_stream_u32(slot + i, PT_EMPTY);
                }
                run += __shfl_sync(0xFFFFFFFFu, inc, 31);
            }
        }
        cnt = warp_sum_u32(cnt);
        if (lane == 0 && cnt) atomicAdd(p.sub_count + sub, cnt);   // the miss and long-piece kernels add theirs
        __syncwarp();                                          // everybody is done with buffer `cur` and the lists
    }
}

// --------------------------------------------------------------------------------------------
// the misses, one piece per lane
// --------------------------------------------------------------------------------------------
static const int MISS_WARPS = 4;
#ifndef MISS_MIN_BLOCKS
#define MISS_MIN_BLOCKS 9
#endif

struct MissSmem {
    uint32_t id[SHORT_MAX * 32];       // [part][lane]
    uint32_t rk[SHORT_MAX * 32];
    uint32_t bytes[4 * 32];            // [word][lane]: the piece bytes, little-endian
};

// Owner election, then a counting sort of the owners by piece length (so that a warp merges pieces of one length):
// dedup with per-block histograms -> bucket bases -> scatter.  Only block-local shared-memory atomics and 18 values per
// block in global memory; no hot global counters.
static const int SORT_BLOCKS_PER_SM = 2;
static const int SORT_THREADS = 1024;                   // dedup / scatter: few blocks (miss_base walks them serially), many threads

__device__ __forceinline__ uint32_t miss_count(const TileParams &p) { return min(p.ctr->n_miss, p.mq.cap); }

// One missed piece per thread.  A piece looks its key up in the memo (a read first: most keys are there already, and a
// read does not serialise on a hot slot the way an atomic does), claims an empty slot with a 128-bit CAS, and takes the
// slot of an equal key as a duplicate.  Winners publish owner[slot]; nobody reads owner[] here, because a duplicate may
// see the key before its owner has published -- the kernel boundary orders that.  Each block may take an equal share of
// half the slots, and stops earlier when the memo does not pay: once it has taken MEMO_TRIAL slots and found fewer than
// one duplicate per 8 slots taken (counted in shared memory, no global counter).  From then on the block's pieces do not read
// their key or probe at all and own themselves, so text whose misses do not repeat pays little more than the length
// histogram.  Owners go to the front of the block's range of `own` and their
// lengths into the block's histogram; duplicates go to the back of the range, for miss_fanout_kernel.
__global__ void __launch_bounds__(SORT_THREADS) miss_dedup_kernel(TileParams p, MissMemo m, unsigned int *block_hist /* [gridDim.x][17] */) {
    __shared__ unsigned int s_h[17], s_n, s_d, s_unplaced, s_won;
    if (threadIdx.x < 17) s_h[threadIdx.x] = 0;
    if (threadIdx.x == 0) { s_n = 0; s_d = 0; s_unplaced = 0; s_won = 0; }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const uint32_t n_miss = (p.ctr->err & ERR_MISSCAP) ? 0u : miss_count(p);
    const uint32_t chunk = (n_miss + gridDim.x - 1) / gridDim.x;
    const uint32_t lo = blockIdx.x * chunk, hi = min(n_miss, lo + chunk);
    const volatile unsigned int *won_so_far = &s_won, *dups_so_far = &s_d;
    for (uint32_t q0 = lo + (threadIdx.x & ~31u); q0 < hi; q0 += SORT_THREADS) {   // warp-uniform trip count: the ballots below
        const uint32_t qi = q0 + lane;
        const bool have = qi < hi;
        const uint32_t taken = *won_so_far;
        const bool full = !m.on || taken >= m.limit || (taken >= MEMO_TRIAL && *dups_so_far * 8u < taken);
        bool dup = false, unplaced = false, won = false;
        uint32_t len = 0;
        if (have) {
            len = p.mq.len[qi];
            if (m.on && len < (uint32_t)SHORT_MAX) {
                unplaced = true;
                if (!full) {
                    const uint4 raw = ld_stream_u4(p.mq.key + qi);
                    U4 k{raw.x, raw.y, raw.z, raw.w};
                    memo_key(k, len);
                    const uint4 kv = make_uint4(k.x, k.y, k.z, k.w);
                    const uint32_t h = memo_hash(k);
                    for (int t = 0; t < MEMO_PROBES; t++) {
                        const uint32_t j = (h + (uint32_t)t) & m.mask;
                        uint4 cur = ld_relaxed_b128(m.key + j);
                        if ((cur.x | cur.y | cur.z | cur.w) == 0u) { cur = cas_zero_b128(m.key + j, kv); won = (cur.x | cur.y | cur.z | cur.w) == 0u; }
                        if (won) { m.owner[j] = qi; unplaced = false; break; }
                        if (cur.x == kv.x && cur.y == kv.y && cur.z == kv.z && cur.w == kv.w) { m.slot[qi] = j; dup = true; unplaced = false; break; }
                    }
                }
            }
        }
        const bool own = have && !dup;
        if (own) atomicAdd(&s_h[len], 1u);
        const uint32_t ob = __ballot_sync(0xFFFFFFFFu, own), db = __ballot_sync(0xFFFFFFFFu, dup);
        const uint32_t ub = __ballot_sync(0xFFFFFFFFu, unplaced), wb = __ballot_sync(0xFFFFFFFFu, won);
        uint32_t bo = 0, bd = 0;
        if (lane == 0) {
            if (ob) bo = atomicAdd(&s_n, (unsigned)__popc(ob));
            if (db) bd = atomicAdd(&s_d, (unsigned)__popc(db));
            if (ub) atomicAdd(&s_unplaced, (unsigned)__popc(ub));
            if (wb) atomicAdd(&s_won, (unsigned)__popc(wb));
        }
        bo = __shfl_sync(0xFFFFFFFFu, bo, 0); bd = __shfl_sync(0xFFFFFFFFu, bd, 0);
        const uint32_t below = (1u << lane) - 1u;
        if (own) m.own[lo + bo + __popc(ob & below)] = qi;
        if (dup) m.own[hi - 1 - (bd + __popc(db & below))] = qi;   // owners + duplicates = hi - lo: the two ends never meet
    }
    __syncthreads();
    if (threadIdx.x < 17) block_hist[blockIdx.x * 17 + threadIdx.x] = s_h[threadIdx.x];
    if (threadIdx.x == 0) {
        m.block_n[2 * blockIdx.x] = s_n; m.block_n[2 * blockIdx.x + 1] = s_d;
        if (s_n) atomicAdd(&p.ctr->n_owner, s_n);
        if (s_unplaced) atomicAdd(&p.ctr->n_unplaced, s_unplaced);
    }
}

// bucket bases: warp l turns column l of block_hist into exclusive offsets (bucket-major, then block order)
__global__ void __launch_bounds__(17 * 32) miss_base_kernel(unsigned int *block_hist, int n_blocks) {
    __shared__ unsigned int s_tot[17];
    const int l = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned int run = 0;
    for (int b0 = 0; b0 < n_blocks; b0 += 32) {
        const int b = b0 + lane;
        const unsigned int c = b < n_blocks ? block_hist[b * 17 + l] : 0u;
        const unsigned int inc = warp_incl_scan_u32(c, lane);
        if (b < n_blocks) block_hist[b * 17 + l] = run + inc - c;
        run += __shfl_sync(0xFFFFFFFFu, inc, 31);
    }
    if (lane == 0) s_tot[l] = run;
    __syncthreads();
    unsigned int base = 0;
    for (int k = 0; k < l; k++) base += s_tot[k];
    for (int b = lane; b < n_blocks; b += 32) block_hist[b * 17 + l] += base;
}

__global__ void __launch_bounds__(SORT_THREADS) miss_scatter_kernel(TileParams p, MissMemo m, const unsigned int *block_base) {
    __shared__ unsigned int s_b[17];
    if (threadIdx.x < 17) s_b[threadIdx.x] = block_base[blockIdx.x * 17 + threadIdx.x];
    __syncthreads();
    const uint32_t n_miss = (p.ctr->err & ERR_MISSCAP) ? 0u : miss_count(p);
    const uint32_t chunk = (n_miss + gridDim.x - 1) / gridDim.x;
    const uint32_t lo = blockIdx.x * chunk, n_own = m.block_n[2 * blockIdx.x];   // the dedup block of the same range
    for (uint32_t k = threadIdx.x; k < n_own; k += SORT_THREADS) {
        const uint32_t qi = m.own[lo + k];
        const uint32_t len = p.mq.len[qi];
        const uint32_t s = atomicAdd(&s_b[len], 1u);
        p.mq.skey[s] = ld_stream_u4(p.mq.key + qi);
        p.mq.smeta[s] = make_uint4(qi, p.mq.roff[qi], p.mq.pos[qi], len);
    }
}

__global__ void __launch_bounds__(MISS_WARPS * 32, MISS_MIN_BLOCKS) miss_kernel(TileParams p, DevTables T) {
    __shared__ MissSmem smem[MISS_WARPS];
    MissSmem &S = smem[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    const uint32_t n_miss = (p.ctr->err & ERR_MISSCAP) ? 0u : p.ctr->n_owner;   // the sorted owners
    const uint32_t stride = gridDim.x * MISS_WARPS * 32;
    for (uint32_t q0 = (blockIdx.x * MISS_WARPS + (threadIdx.x >> 5)) * 32; q0 < n_miss; q0 += stride) {
        const bool have = q0 + lane < n_miss;
        uint4 key = make_uint4(0, 0, 0, 0), meta = make_uint4(0, 0, 0, 0);
        if (have) { key = ld_stream_u4(p.mq.skey + q0 + lane); meta = ld_stream_u4(p.mq.smeta + q0 + lane); }
        const int len = (int)meta.w;
        S.bytes[0 * 32 + lane] = key.x; S.bytes[1 * 32 + lane] = key.y; S.bytes[2 * 32 + lane] = key.z; S.bytes[3 * 32 + lane] = key.w;
        const int n_max = (int)__reduce_max_sync(0xFFFFFFFFu, (unsigned)len);
        SmemCol32 id{S.id + lane}, rk{S.rk + lane};
        const uint32_t *bw = S.bytes + lane;
        const uint32_t mask = merge_short_conv(
            T, [&](int j) { return (bw[(j >> 2) * 32] >> (8 * (j & 3))) & 0xFFu; }, len, n_max, 0xFFFFFFFFu, id, rk);
        if (have) {
            // the result record the gather reads: count + the first three tokens (94 % of the missed pieces end as <= 3
            // tokens); longer results also go to mres.  One 16-byte store per piece instead of a token array + a count.
            const uint32_t c = (uint32_t)__popc(mask);
            uint32_t t[3] = {0, 0, 0}, k = 0; bool bad = false;
            uint32_t *dst = p.mres + meta.y;
            for (uint32_t mm = mask; mm; k++) {
                const int j = __ffs(mm) - 1; mm &= mm - 1;
                const uint32_t x = id[j];
                bad |= x >= PSEUDO_BASE;
                if (k == 0) t[0] = x; else if (k == 1) t[1] = x; else if (k == 2) t[2] = x;
                if (c > 3) dst[k] = x;
            }
            if (bad) atomicOr(&p.ctr->err, ERR_NOBYTE);
            st_stream_u4(p.mq.rec + meta.x, make_uint4(c, t[0], t[1], t[2]));
            atomicAdd(&p.sub_count[meta.z >> 10], c);
        }
        __syncwarp();
    }
}

// One duplicate per thread, from the back of its dedup block's range of `own` (same grid): it takes its owner's record
// and result region and credits the tokens to its sub-tile (one atomic per run of lanes in the same sub-tile: the probe
// queues a sub-tile's misses back to back).  Owners credited theirs in miss_kernel.
__global__ void __launch_bounds__(SORT_THREADS) miss_fanout_kernel(TileParams p, MissMemo m) {
    const int lane = threadIdx.x & 31;
    const uint32_t n_miss = (p.ctr->err & ERR_MISSCAP) ? 0u : miss_count(p);
    const uint32_t chunk = (n_miss + gridDim.x - 1) / gridDim.x;
    const uint32_t hi = min(n_miss, blockIdx.x * chunk + chunk), n_dup = m.block_n[2 * blockIdx.x + 1];
    for (uint32_t k0 = threadIdx.x & ~31u; k0 < n_dup; k0 += SORT_THREADS) {   // warp-uniform: the match below
        const uint32_t k = k0 + lane;
        uint32_t c = 0, sub = 0xFFFFFFFFu;
        if (k < n_dup) {
            const uint32_t qi = m.own[hi - 1 - k];
            const uint32_t o = m.owner[m.slot[qi]];
            const uint4 r = p.mq.rec[o];
            p.mq.rec[qi] = r;
            if (r.x > 3) p.mq.roff[qi] = p.mq.roff[o];
            c = r.x;
            sub = p.mq.pos[qi] >> 10;
        }
        const uint32_t same = __match_any_sync(0xFFFFFFFFu, sub);
        const uint32_t sum = __reduce_add_sync(same, c);
        if (sub != 0xFFFFFFFFu && lane == __ffs(same) - 1 && sum) atomicAdd(&p.sub_count[sub], sum);
    }
}

static const int SCAN_ITEMS = 4096;                 // counts per block of the two-level scan

__global__ void __launch_bounds__(256) scan_partial_kernel(const uint32_t *__restrict__ cnt, long long n,
                                                          unsigned long long *__restrict__ part) {
    __shared__ unsigned long long s_w[8];
    const long long lo = (long long)blockIdx.x * SCAN_ITEMS;
    unsigned long long sum = 0;
    for (int k = threadIdx.x; k < SCAN_ITEMS; k += 256) { long long i = lo + k; if (i < n) sum += cnt[i]; }
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) { unsigned long long t = 0; for (int i = 0; i < 8; i++) t += s_w[i]; part[blockIdx.x] = t; }
}

// single block: exclusive scan of the per-block partial sums (n_blocks <= a few thousand)
__global__ void __launch_bounds__(1024) scan_top_kernel(unsigned long long *part, long long n_blocks, Counters *ctr) {
    __shared__ unsigned long long s_part[1024];
    const int tid = threadIdx.x;
    const long long per = (n_blocks + 1023) / 1024;
    const long long lo = tid * per, hi = (lo + per < n_blocks) ? lo + per : n_blocks;
    unsigned long long sum = 0;
    for (long long i = lo; i < hi; i++) sum += part[i];
    s_part[tid] = sum;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        unsigned long long v = (tid >= o) ? s_part[tid - o] : 0ull;
        __syncthreads();
        s_part[tid] += v;
        __syncthreads();
    }
    unsigned long long run = s_part[tid] - sum;
    for (long long i = lo; i < hi; i++) { unsigned long long c = part[i]; part[i] = run; run += c; }
    if (tid == 1023) ctr->total_tokens = s_part[1023];
}

__global__ void __launch_bounds__(256) scan_final_kernel(const uint32_t *__restrict__ cnt, long long n,
                                                        const unsigned long long *__restrict__ part,
                                                        unsigned long long *__restrict__ base, const Counters *ctr) {
    __shared__ unsigned long long s_w[8];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const long long lo = (long long)blockIdx.x * SCAN_ITEMS + (long long)tid * 16;   // 16 consecutive counts per thread
    uint32_t c[16]; unsigned long long sum = 0;
#pragma unroll
    for (int k = 0; k < 16; k++) { long long i = lo + k; c[k] = (i < n) ? cnt[i] : 0u; sum += c[k]; }
    unsigned long long inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    unsigned long long run = part[blockIdx.x] + inc - sum;
    for (int i = 0; i < wid; i++) run += s_w[i];
#pragma unroll
    for (int k = 0; k < 16; k++) { long long i = lo + k; if (i < n) base[i] = run; run += c[k]; }
    if (blockIdx.x == 0 && tid == 0) base[n] = ctr->total_tokens;
}

// chunked host path: rebase a slice of the caller's document offsets / globalise token offsets
__global__ void add_offset_kernel(unsigned long long *a, unsigned long long n, long long delta) {
    unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (i < n) a[i] = (unsigned long long)((long long)a[i] + delta);
}

// --------------------------------------------------------------------------------------------
// gather.  One warp per sub-tile, piece-parallel: a step takes 32 consecutive slots of ptok (coalesced), turns them
// into token counts (hit 1, miss / long piece: looked up), scans them across the warp and writes the tokens at
// base + prefix.  Per-document token offsets: a document start coincides with a piece start, so its offset is the
// token prefix of that piece (kept in shared memory only for sub-tiles that contain a document start).
// --------------------------------------------------------------------------------------------
static const int GATHER_WARPS = 8;

// MODE 0: every sub-tile, those with a document start skipped (no shared memory, 32 registers: full occupancy);
// MODE 1: the sub-tiles of the doc-tile list (sparse documents: a few thousand of a million sub-tiles);
// MODE 2: every sub-tile, all treated as holding document starts (dense documents: the list would be the whole grid).
// MODE 1 / 2 keep 4 KiB of per-piece token prefixes per warp in shared memory.
template <int MODE>
__global__ void __launch_bounds__(GATHER_WARPS * 32, MODE ? 6 : 8) gather_kernel(TileParams p) {
    constexpr bool DOCS = MODE != 0;
    __shared__ uint32_t s_pref[DOCS ? GATHER_WARPS : 1][DOCS ? SUB_BYTES + 1 : 1];
    const int lane = threadIdx.x & 31, warp = DOCS ? (threadIdx.x >> 5) : 0;
    long long sub = (long long)blockIdx.x * GATHER_WARPS + (threadIdx.x >> 5);
    if (MODE == 1) {
        if (sub >= (long long)p.ctr->n_doc_tiles) return;
        sub = (long long)p.doc_tiles[sub];
    }
    if (sub >= p.n_sub) return;
    const unsigned long long base = p.sub_base[sub];
    const uint32_t *slot = p.ptok + sub * SUB_BYTES;
    const long long sub_byte = sub * SUB_BYTES;
    const long long gw = sub * 32 + lane;
    const bool in = gw < p.n_words;
    const uint32_t dm = in ? ld_stream_u32(p.dbits + gw) : 0u;
    uint32_t pv = in ? ld_stream_u32(p.pbits + gw) : 0u;
    {
        const long long span0 = sub_byte + lane * 32;
        if (span0 + 32 > p.n_bytes) {
            const long long keep = p.n_bytes - span0;
            pv = keep <= 0 ? 0u : (pv & ((1u << keep) - 1u));
        }
    }
    const uint32_t c = __popc(pv);
    const uint32_t pinc = warp_incl_scan_u32(c, lane);
    const uint32_t pi0 = pinc - c;                           // index of this lane's first piece
    const uint32_t np = __shfl_sync(0xFFFFFFFFu, pinc, 31);
    if (MODE == 0 && __any_sync(0xFFFFFFFFu, dm != 0)) return;           // a document starts here: MODE 1 takes this sub-tile
    uint32_t run = 0;                                        // tokens of the sub-tile so far
    // Software pipeline over steps of 32 pieces: the slot load of step t+2 and the count look-up of step t+1 (misses and
    // long pieces only) are in flight while step t is scanned and written, so a step does not wait for L2 twice.
    auto load_slot = [&](uint32_t i0) -> uint32_t { const uint32_t i = i0 + lane; return i < np ? ld_stream_u32(slot + i) : PT_EMPTY; };
    auto count_of = [&](uint32_t v) -> uint32_t {
        if (v == PT_EMPTY) return 0u;
        const uint32_t kind = v & PT_KIND, qi = v & PT_PAYLOAD;
        return kind == 0 ? 1u : kind == PT_MISS ? __ldg(reinterpret_cast<const uint32_t *>(p.mq.rec + qi)) : p.q.ntok[qi];
    };
    uint32_t v0 = load_slot(0), v1 = load_slot(32);
    uint32_t n0 = count_of(v0);
    for (uint32_t i0 = 0; i0 < np; i0 += 32) {
        const uint32_t v2 = load_slot(i0 + 64);              // step t+2: slot
        const uint32_t n1 = count_of(v1);                    // step t+1: count
        const uint32_t i = i0 + lane, v = v0, n = n0;
        const uint32_t kind = v & PT_KIND, qi = v & PT_PAYLOAD;
        const uint32_t incl = warp_incl_scan_u32(n, lane);
        const uint32_t excl = incl - n;
        const unsigned long long k = base + run + excl;
        if (DOCS && i < np) s_pref[warp][i] = run + excl;
        unsigned long long lsrc = 0;
        if (n) {
            if (kind == 0) st_stream_u32(p.out + k, v);
            else if (kind == PT_MISS) {                               // the record is in the sector its count came from
                const uint4 r = __ldg(p.mq.rec + qi);
                st_stream_u32(p.out + k, r.y);
                if (n > 1) st_stream_u32(p.out + k + 1, r.z);
                if (n > 2) st_stream_u32(p.out + k + 2, r.w);
                if (n > 3) { const uint32_t *src = p.mres + p.mq.roff[qi]; for (uint32_t x = 3; x < n; x++) st_stream_u32(p.out + k + x, src[x]); }
            }
            else {
                lsrc = p.q.start[qi];
                if (n <= 32) for (uint32_t x = 0; x < n; x++) st_stream_u32(p.out + k + x, p.ltok[lsrc + x]);
            }
        }
        // long pieces with more than 32 tokens: copied by the whole warp, giant ones left to the whole grid
        for (uint32_t pending = __ballot_sync(0xFFFFFFFFu, v != PT_EMPTY && kind == PT_LONG && n > 32); pending; pending &= pending - 1) {
            const int src_lane = __ffs(pending) - 1;
            const unsigned long long dst = __shfl_sync(0xFFFFFFFFu, k, src_lane);
            const unsigned long long bs = __shfl_sync(0xFFFFFFFFu, lsrc, src_lane);
            const uint32_t nt = __shfl_sync(0xFFFFFFFFu, n, src_lane);
            if (nt > 4096) {
                if (lane == 0) { const uint32_t e = atomicAdd(&p.ctr->n_big, 1u); p.big_dst[e] = dst; p.big_src[e] = bs; p.big_n[e] = nt; }
                continue;
            }
            for (uint32_t x = lane; x < nt; x += 32) st_stream_u32(p.out + dst + x, p.ltok[bs + x]);
        }
        run += __shfl_sync(0xFFFFFFFFu, incl, 31);
        v0 = v1; v1 = v2; n0 = n1;
    }
    if (DOCS) {
        __syncwarp();
        if (dm) {
            unsigned long long d = (unsigned long long)__ldg(p.span_first_doc + gw);
            for (uint32_t walk = dm; walk; walk &= walk - 1) {
                const int j = __ffs(walk) - 1;
                const unsigned long long pos = (unsigned long long)(sub_byte + lane * 32 + j);
                const uint32_t pidx = pi0 + __popc(pv & ((1u << j) - 1u));
                const unsigned long long tok = base + (pidx < np ? s_pref[warp][pidx] : run);
                while (d <= p.n_docs && p.doc_off[d] == pos) { p.tok_off[d] = tok; d++; }
            }
        }
    }
}

// token copies of giant pieces, spread over the whole grid
__global__ void __launch_bounds__(256) big_copy_kernel(TileParams p) {
    const unsigned int nb = p.ctr->n_big;
    for (unsigned int e = 0; e < nb; e++) {
        const unsigned long long dst = p.big_dst[e], src = p.big_src[e];
        const uint32_t n = p.big_n[e];
        for (unsigned long long x = blockIdx.x * 256ull + threadIdx.x; x < n; x += (unsigned long long)gridDim.x * 256ull)
            p.out[dst + x] = p.ltok[src + x];
    }
}
