// kernels_train.cuh -- BPE vocabulary training on the device (tiktoken/_educational.py `bpe_train`).
//
// Words are the regex pieces of the corpus (pre-tokeniser of kernels_pretok.cuh, chunk by chunk).  Identical pieces
// have identical states, so the trainer works on the distinct pieces ("words") in order of first appearance, each
// weighted by its count.  Layout after the distinct-word stage:
//   sym[woff[w] .. woff[w] + wlen[w])  the symbol ids of word w (ids 0..255 are the bytes), then TR_SENT; the slots a
//                                      word frees when it shrinks become TR_SENT too, so a flat scan of sym sees
//                                      exactly the adjacent pairs of the words
//   pair table                         open addressing (left << 32 | right) -> weighted count, plus the list of
//                                      occupied slots (the max scan reads only those)
// One merge step is five kernels with no host synchronisation (the host replays a CUDA graph of many steps):
//   max     highest count over the occupied pair slots
//   first   the first flat position (= first word, then first position: rule of the reference's Counter + max())
//           whose pair has that count; blocks stride over tiles in order and stop past the best position found
//   commit  one thread: the merged token's id (an existing id when its bytes already have one: polynomial hash of
//           the bytes, h(a|b) = h(a) B^|b| + h(b)), the merge record, the next step's reset
//   mark    flat scan for the winner; each word that contains it is listed once
//   apply   warp per listed word: left-to-right merge without overlap, in place; the pair counts change only
//           around merged positions: the old pairs that touch one are subtracted, the new pairs that touch a
//           merged symbol are added (both times the word's weight)
#pragma once
#include "dev_common.cuh"

namespace b2bpe {

static const uint32_t TR_SENT = 0xFFFFFFFFu;
static const unsigned long long TR_EMPTY = ~0ull;
static const unsigned long long TR_B = 0x100000001B3ull;      // polynomial base (odd) of the byte-string hashes
static const uint32_t TR_RUN = 0, TR_DONE = 1, TR_NOPAIR = 2, TR_CAP = 3, TR_INTERNAL = 4;

struct TrainState {            // device-resident; the host reads it once per graph batch
    unsigned long long max, best;
    uint32_t L, R, id;         // the current step's merge
    uint32_t n_ids;            // 256 + merges whose bytes were new (= len(ranks) of the reference)
    uint32_t n_merges, stop, n_aff, n_occ, err, pad;
};

struct TrainWords {            // piece hash table of the distinct-word stage (key 0 = empty)
    unsigned long long *key, *cnt, *first; uint32_t *len;
    unsigned long long mask;
    unsigned long long *n_used;
};

struct TrainPairs { unsigned long long *key, *cnt; uint32_t *occ; unsigned long long mask; };

struct TrainTok {              // per token id: hash, B^len, length; (hash, length) -> id
    unsigned long long *h, *pw, *len; uint32_t *slot; unsigned long long mask;
};

__device__ __forceinline__ unsigned long long tr_mix(unsigned long long k) {
    k ^= k >> 33; k *= 0xFF51AFD7ED558CCDull; k ^= k >> 33; k *= 0xC4CEB9FE1A85EC53ull; k ^= k >> 33;
    return k;
}

// ---- distinct words ------------------------------------------------------------------------------------------------
// Every piece of a chunk: one thread per 32-bit word of the piece-start bitmask, fn(start, end) per piece.  A piece
// ends at the next piece start; the end-of-text sentinel bit bounds the walk.
template <class F>
__device__ __forceinline__ void tr_for_pieces(const uint32_t *pbits, long long n_bytes, long long w, F fn) {
    uint32_t word = pbits[w];
    while (word) {
        const int j = __ffs(word) - 1;
        word &= word - 1;
        const long long p = w * 32 + j;
        if (p >= n_bytes) return;
        long long e;
        if (word) e = w * 32 + __ffs(word) - 1;
        else {
            long long v = w + 1;
            while (!pbits[v]) v++;
            e = v * 32 + __ffs(pbits[v]) - 1;
        }
        fn(p, e);
    }
}

__device__ __forceinline__ unsigned long long tr_piece_key(const uint8_t *t, long long p, long long e) {
    unsigned long long h = 0;
    for (long long i = p; i < e; i++) h = h * TR_B + (unsigned long long)t[i] + 1ull;
    unsigned long long k = tr_mix(h ^ ((unsigned long long)(e - p) * 0x9E3779B97F4A7C15ull));
    return k ? k : 1ull;
}

__global__ void train_count_kernel(const uint32_t *__restrict__ pbits, long long n_bytes, long long n_words,
                                   unsigned long long *n_pieces) {
    const long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    uint32_t c = 0;
    if (w < n_words) {
        uint32_t word = pbits[w];
        const long long lim = n_bytes - w * 32;               // positions >= n_bytes hold no piece start
        if (lim < 32) word &= lim <= 0 ? 0u : (1u << lim) - 1u;
        c = (uint32_t)__popc(word);
    }
    c = __reduce_add_sync(0xFFFFFFFFu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(n_pieces, (unsigned long long)c);
}

__device__ __forceinline__ unsigned long long tr_word_slot(const TrainWords &W, unsigned long long k) {
    unsigned long long h = tr_mix(k) & W.mask;
    for (;;) {
        const unsigned long long old = atomicCAS(&W.key[h], 0ull, k);
        if (old == 0ull) { atomicAdd(W.n_used, 1ull); return h; }
        if (old == k) return h;
        h = (h + 1) & W.mask;
    }
}

__global__ void train_insert_kernel(const uint8_t *__restrict__ text, long long n_bytes, const uint32_t *__restrict__ pbits,
                                    long long n_words, unsigned long long base, TrainWords W) {
    const long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (w >= n_words) return;
    tr_for_pieces(pbits, n_bytes, w, [&](long long p, long long e) {
        const unsigned long long s = tr_word_slot(W, tr_piece_key(text, p, e));
        atomicAdd(&W.cnt[s], 1ull);
        atomicMin(&W.first[s], base + (unsigned long long)p);
        W.len[s] = (uint32_t)(e - p);
    });
}

// After a chunk's inserts the first occurrence of each of its pieces is final (chunks go in corpus order): every
// piece compares its bytes with that occurrence (a hash collision fails the call, never merges two words), and the
// first occurrences set their bit in fbits (bit = corpus byte offset).
__global__ void train_verify_kernel(const uint8_t *__restrict__ text, long long n_bytes, const uint32_t *__restrict__ pbits,
                                    long long n_words, unsigned long long base, TrainWords W, const uint8_t *__restrict__ all,
                                    uint32_t *fbits, TrainState *st) {
    const long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (w >= n_words) return;
    tr_for_pieces(pbits, n_bytes, w, [&](long long p, long long e) {
        const unsigned long long k = tr_piece_key(text, p, e);
        unsigned long long h = tr_mix(k) & W.mask;
        while (W.key[h] != k) h = (h + 1) & W.mask;
        const unsigned long long f = W.first[h], g = base + (unsigned long long)p;
        if (f == g) { atomicOr(&fbits[g >> 5], 1u << (g & 31)); return; }
        bool same = W.len[h] == (uint32_t)(e - p);
        for (long long i = 0; same && i < e - p; i++) same = all[f + i] == text[p + i];
        if (!same) atomicOr(&st->err, 1u);
    });
}

// grow the piece table: re-insert every occupied slot
__global__ void train_rehash_kernel(TrainWords O, unsigned long long n_old, TrainWords N) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n_old;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = O.key[i];
        if (!k) continue;
        const unsigned long long s = tr_word_slot(N, k);
        N.cnt[s] = O.cnt[i]; N.first[s] = O.first[i]; N.len[s] = O.len[i];
    }
}

// first-occurrence bits per 1 KiB of corpus (for the word index = rank of the first occurrence)
__global__ void train_tile_count_kernel(const uint32_t *__restrict__ fbits, long long n_tiles, uint32_t *tcnt) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= n_tiles) return;
    uint32_t c = 0;
    for (int j = 0; j < 32; j++) c += (uint32_t)__popc(fbits[t * 32 + j]);
    tcnt[t] = c;
}

__global__ void train_compact_kernel(TrainWords W, const uint32_t *__restrict__ fbits, const unsigned long long *__restrict__ tbase,
                                     unsigned long long *wfirst, uint32_t *wlen, unsigned long long *wcnt, uint32_t *wl1,
                                     unsigned long long n_words, TrainState *st) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i <= W.mask;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        if (!W.key[i]) continue;
        const unsigned long long f = W.first[i];
        unsigned long long idx = tbase[f >> 10];
        for (unsigned long long j = (f >> 10) * 32; j < (f >> 5); j++) idx += (unsigned long long)__popc(fbits[j]);
        idx += (unsigned long long)__popc(fbits[f >> 5] & ((1u << (f & 31)) - 1u));
        if (idx >= n_words) { atomicOr(&st->err, 2u); continue; }
        wfirst[idx] = f; wlen[idx] = W.len[i]; wcnt[idx] = W.cnt[i]; wl1[idx] = W.len[i] + 1u;
    }
}

// warp per word: its bytes as symbol ids, then the separator
__global__ void train_fill_kernel(const uint8_t *__restrict__ all, const unsigned long long *__restrict__ wfirst,
                                  const uint32_t *__restrict__ wlen, const unsigned long long *__restrict__ woff,
                                  unsigned long long n_words, uint32_t *sym) {
    const int lane = threadIdx.x & 31;
    for (unsigned long long w = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5; w < n_words;
         w += ((unsigned long long)gridDim.x * blockDim.x) >> 5) {
        const unsigned long long f = wfirst[w], o = woff[w];
        const uint32_t n = wlen[w];
        for (uint32_t j = lane; j < n; j += 32) sym[o + j] = all[f + j];
        if (lane == 0) sym[o + n] = TR_SENT;
    }
}

// ---- pair table ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long tr_pair_key(uint32_t a, uint32_t b) { return (unsigned long long)a << 32 | b; }

__device__ __forceinline__ unsigned long long tr_pair_get(const TrainPairs &P, unsigned long long k) {
    unsigned long long h = tr_mix(k) & P.mask;
    for (unsigned long long n = 0; n <= P.mask; n++) {
        const unsigned long long x = P.key[h];
        if (x == k) return P.cnt[h];
        if (x == TR_EMPTY) return 0ull;
        h = (h + 1) & P.mask;
    }
    return 0ull;
}

__device__ __forceinline__ void tr_pair_add(const TrainPairs &P, unsigned long long k, unsigned long long d, TrainState *st) {
    unsigned long long h = tr_mix(k) & P.mask;
    for (unsigned long long n = 0; n <= P.mask; n++) {
        unsigned long long x = *(volatile unsigned long long *)&P.key[h];
        if (x == TR_EMPTY) {
            x = atomicCAS(&P.key[h], TR_EMPTY, k);
            if (x == TR_EMPTY) { P.occ[atomicAdd(&st->n_occ, 1u)] = (uint32_t)h; x = k; }
        }
        if (x == k) { atomicAdd(&P.cnt[h], d); return; }
        h = (h + 1) & P.mask;
    }
    atomicOr(&st->err, 4u);                    // table full: sized so that it cannot happen (DESIGN §3.4d)
}

// warp per word: every adjacent pair, times the word's weight
__global__ void train_pairs_init_kernel(const uint32_t *__restrict__ sym, const unsigned long long *__restrict__ woff,
                                        const uint32_t *__restrict__ wlen, const unsigned long long *__restrict__ wcnt,
                                        unsigned long long n_words, TrainPairs P, TrainState *st) {
    const int lane = threadIdx.x & 31;
    for (unsigned long long w = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5; w < n_words;
         w += ((unsigned long long)gridDim.x * blockDim.x) >> 5) {
        const uint32_t *s = sym + woff[w];
        const uint32_t n = wlen[w];
        const unsigned long long c = wcnt[w];
        for (uint32_t j = lane; j + 1 < n; j += 32) tr_pair_add(P, tr_pair_key(s[j], s[j + 1]), c, st);
    }
}

// token ids 0..255 = the single bytes: hash b + 1, B^1, length 1
__global__ void train_tok_init_kernel(TrainTok T) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    for (uint32_t b = 0; b < 256; b++) {
        T.h[b] = b + 1ull; T.pw[b] = TR_B; T.len[b] = 1ull;
        unsigned long long s = tr_mix((b + 1ull) ^ 0x9E3779B97F4A7C15ull) & T.mask;
        while (T.slot[s] != TR_SENT) s = (s + 1) & T.mask;
        T.slot[s] = b;
    }
}

// ---- one merge step --------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) { const unsigned long long y = __shfl_xor_sync(0xFFFFFFFFu, v, o); v = y > v ? y : v; }
    return v;
}
__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) { const unsigned long long y = __shfl_xor_sync(0xFFFFFFFFu, v, o); v = y < v ? y : v; }
    return v;
}

__global__ void __launch_bounds__(256) train_max_kernel(TrainPairs P, TrainState *st) {
    if (st->stop) return;
    const uint32_t n = st->n_occ;
    unsigned long long m = 0;
    for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u) {
        const unsigned long long c = P.cnt[P.occ[i]];
        m = c > m ? c : m;
    }
    m = warp_max_u64(m);
    if ((threadIdx.x & 31) == 0 && m) atomicMax(&st->max, m);
}

static const int TR_FIRST_ITEMS = 8;

__global__ void __launch_bounds__(256) train_first_kernel(const uint32_t *__restrict__ sym, unsigned long long n_sym,
                                                          TrainPairs P, TrainState *st) {
    __shared__ int s_go;
    __shared__ unsigned long long s_min[8];
    if (st->stop) return;
    const unsigned long long mx = st->max;
    if (mx == 0) return;
    const unsigned long long tile = 256ull * TR_FIRST_ITEMS;
    for (unsigned long long t = blockIdx.x; t * tile < n_sym; t += gridDim.x) {
        const unsigned long long base = t * tile;
        if (threadIdx.x == 0) s_go = base <= *(volatile unsigned long long *)&st->best;
        __syncthreads();
        if (!s_go) return;                     // a pair of this count occurs earlier: nothing past it matters
        unsigned long long mine = ~0ull;
        for (int k = 0; k < TR_FIRST_ITEMS && mine == ~0ull; k++) {
            const unsigned long long p = base + (unsigned long long)k * 256 + threadIdx.x;
            if (p + 1 < n_sym) {
                const uint32_t a = sym[p], b = sym[p + 1];
                if (a != TR_SENT && b != TR_SENT && tr_pair_get(P, tr_pair_key(a, b)) == mx) mine = p;
            }
        }
        mine = warp_min_u64(mine);
        if ((threadIdx.x & 31) == 0) s_min[threadIdx.x >> 5] = mine;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long m = s_min[0];
            for (int i = 1; i < 8; i++) m = s_min[i] < m ? s_min[i] : m;
            if (m != ~0ull) atomicMin(&st->best, m);
        }
        __syncthreads();
    }
}

__global__ void train_commit_kernel(const uint32_t *__restrict__ sym, TrainTok T, uint32_t *merges, uint32_t merge_cap,
                                    uint32_t vocab_size, TrainState *st) {
    if (threadIdx.x != 0 || blockIdx.x != 0 || st->stop) return;
    if (st->err) { st->stop = TR_INTERNAL; return; }
    if (st->max == 0) { st->stop = TR_NOPAIR; return; }
    if (st->best == ~0ull) { st->stop = TR_INTERNAL; return; }
    if (st->n_merges >= merge_cap) { st->stop = TR_CAP; return; }
    const uint32_t L = sym[st->best], R = sym[st->best + 1];
    const unsigned long long h = T.h[L] * T.pw[R] + T.h[R], len = T.len[L] + T.len[R];
    unsigned long long s = tr_mix(h ^ (len * 0x9E3779B97F4A7C15ull)) & T.mask;
    uint32_t id = TR_SENT;
    for (;;) {
        const uint32_t v = T.slot[s];
        if (v == TR_SENT) break;
        if (T.h[v] == h && T.len[v] == len) { id = v; break; }    // the bytes already have an id (the host checks the bytes)
        s = (s + 1) & T.mask;
    }
    if (id == TR_SENT) {
        id = st->n_ids++;
        T.h[id] = h; T.pw[id] = T.pw[L] * T.pw[R]; T.len[id] = len; T.slot[s] = id;
    }
    const uint32_t m = st->n_merges++;
    merges[3 * m] = L; merges[3 * m + 1] = R; merges[3 * m + 2] = id;
    st->L = L; st->R = R; st->id = id;
    st->max = 0; st->best = ~0ull; st->n_aff = 0;
    if (st->n_ids >= vocab_size) st->stop = TR_DONE;
}

__global__ void __launch_bounds__(256) train_mark_kernel(const uint32_t *__restrict__ sym, unsigned long long n_sym,
                                                         const unsigned long long *__restrict__ woff, unsigned long long n_words,
                                                         uint32_t *stamp, uint32_t *aff, TrainState *st) {
    if (st->stop) return;
    const uint32_t L = st->L, R = st->R, tag = st->n_merges;
    for (unsigned long long p = blockIdx.x * 256ull + threadIdx.x; p + 1 < n_sym; p += gridDim.x * 256ull) {
        if (sym[p] != L || sym[p + 1] != R) continue;
        unsigned long long lo = 0, hi = n_words;             // last word with woff <= p
        while (hi - lo > 1) { const unsigned long long mid = (lo + hi) >> 1; if (woff[mid] <= p) lo = mid; else hi = mid; }
        if (atomicExch(&stamp[lo], tag) != tag) aff[atomicAdd(&st->n_aff, 1u)] = (uint32_t)lo;
    }
}

__global__ void __launch_bounds__(256) train_apply_kernel(uint32_t *sym, const unsigned long long *__restrict__ woff,
                                                          uint32_t *wlen, const unsigned long long *__restrict__ wcnt,
                                                          const uint32_t *__restrict__ aff, TrainPairs P, TrainState *st) {
    if (st->stop) return;
    const uint32_t L = st->L, R = st->R, NEW = st->id, n_aff = st->n_aff;
    const int lane = threadIdx.x & 31;
    for (uint32_t k = (blockIdx.x * 256u + threadIdx.x) >> 5; k < n_aff; k += (gridDim.x * 256u) >> 5) {
        const uint32_t w = aff[k];
        uint32_t *sp = sym + woff[w];
        const uint32_t n = wlen[w];
        const unsigned long long wt = wcnt[w], nwt = 0ull - wt;
        uint32_t carry = 0, out = 0;                     // carry: the last symbol of the previous tile starts a merge
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t i = base + lane;
            const uint32_t x0 = i < n ? sp[i] : TR_SENT, x1 = i + 1 < n ? sp[i + 1] : TR_SENT;
            const uint32_t x2 = i + 2 < n ? sp[i + 2] : TR_SENT, x3 = i + 3 < n ? sp[i + 3] : TR_SENT;
            const uint32_t M = __ballot_sync(0xFFFFFFFFu, x0 == L && x1 == R);
            const uint32_t E = __shfl_sync(0xFFFFFFFFu, (uint32_t)(x1 == L && x2 == R) | (uint32_t)(x2 == L && x3 == R) << 1, 31);
            const unsigned long long M64 = (unsigned long long)M | (unsigned long long)E << 32;   // matches at base .. base+33
            // merge starts: a[j] = m[j] && !a[j-1]; two different symbols cannot overlap, so then a == m
            unsigned long long A = M64;
            if (L == R) {
                A = 0; unsigned long long prev = carry;
                for (int j = 0; j < 34; j++) { const unsigned long long b = (M64 >> j) & ~prev & 1ull; A |= b << j; prev = b; }
            }
            const unsigned long long C = (A << 1) | carry;  // bit j: symbol base+j is the right half of a merge
            const unsigned long long Pm = A | C;            // bit j: symbol base+j takes part in a merge
            const uint32_t a_i = (uint32_t)(A >> lane) & 1u, c_i = (uint32_t)(C >> lane) & 1u;
            if (i + 1 < n && ((Pm >> lane) & 3ull)) tr_pair_add(P, tr_pair_key(x0, x1), nwt, st);   // old pair touches a merge
            const bool emit = i < n && !c_i;
            const uint32_t v = a_i ? NEW : x0;
            if (emit) {
                const uint32_t nx = a_i ? i + 2 : i + 1;           // the next symbol that survives
                if (nx < n) {
                    const uint32_t a_n = (uint32_t)(A >> (nx - base)) & 1u;
                    const uint32_t r = a_n ? NEW : (a_i ? x2 : x1);
                    if (a_i | a_n) tr_pair_add(P, tr_pair_key(v, r), wt, st);               // new pair touches a merge
                }
            }
            const uint32_t EM = __ballot_sync(0xFFFFFFFFu, emit);
            __syncwarp();                                          // every read of this tile precedes the writes
            if (emit) sp[out + __popc(EM & ((1u << lane) - 1u))] = v;
            out += (uint32_t)__popc(EM);
            carry = (uint32_t)(A >> 31) & 1u;
            __syncwarp();
        }
        for (uint32_t j = out + lane; j < n; j += 32) sp[j] = TR_SENT;
        if (lane == 0) wlen[w] = out;
    }
}

}  // namespace b2bpe
