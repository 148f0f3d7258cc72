// b200bpe.cu -- the engine and the C ABI of libb200bpe.so (see include/b200bpe.h).  sm_90a only.
//
// Path replaced: CoreBPE::encode_ordinary / CoreBPE::encode (src/lib.rs:360-442) and the per-call
// thread pool that fans documents out to it (tiktoken/core.py:164-206).  One call encodes the
// whole batch (kernels in kernels_*.cuh):
//
//   mark_docs_kernel      doc_off[] -> doc-start bitmask D + first-doc-per-span index
//   special_*_kernel      (CoreBPE::encode only) multi-pattern scan: disallowed specials -> error; allowed specials ->
//                         haystack boundaries, interior mask, special-piece mask + their ids
//   pretok_kernel<PAT>    UTF-8 bytes + D -> piece-start bitmask P   (bit-parallel regex rules)
//   find_long_kernel      P -> queue of pieces longer than 16 bytes + one work list per length class
//   mid_group{16,32}_kernel  17..128 bytes: a group of lanes per piece, merge state in shared memory
//   pmerge{,_long}_kernel    129..1024 bytes: a warp per piece, a few rounds of parallel merges
//                         (ranks of 2^22 and above: mid_thread_kernel 17..256 bytes, a piece per lane, and
//                         long_piece_kernel 257..1024 bytes, a warp per piece)
//   long_piece_kernel     1025..4096 bytes: a warp per piece;  giant_piece_kernel ..32768 bytes: a block per piece;
//   cluster_piece_kernel  beyond: a thread-block cluster (8 x 1024 threads, DSMEM carries) per piece
//                         -- the round-synchronous exact merge in global scratch
//   probe_kernel          persistent warps, TMA-staged 1 KiB sub-tiles: whole-piece table probe of every short piece
//                         (one 32 B sector each), one slot per piece, misses -> global queue with their key bytes
//   miss_{dedup,base,scatter}, miss_kernel, miss_fanout   the ~5 % misses: one owner per distinct piece (a per-call
//                         memo), owners sorted by length, one piece per lane, warp-convergent exact min-rank merge on
//                         dense records, the owner's result copied to every other occurrence
//   scan_{partial,top,final}, gather_kernel, big_copy_kernel   token counts -> offsets -> tokens and
//                         per-document offsets at their final place
//   utf8_check, bytes_*   (bytes mode only, kernels_bytes.cuh) documents that are not well-formed UTF-8: cut at the
//                         first ill-formed byte, repair of the last piece, a second run over the unstable pieces, splice
//   unstable_*            (completion search only, kernels_unstable.cuh) the unstable tail of every document, the tokens
//                         that could continue it, run 2 over the candidates in rounds, truncation and deduplication
//
// No tensor cores: nothing here is a contraction.  The work is byte/integer, bound by HBM reads
// of the text, L2 probes of the rank tables and instruction issue.
//
// Host side: one DevCtx per CUDA device (tables replicated, three pipeline slots each); batches are cut at
// document boundaries, and documents larger than a chunk at seams (doc_seams.h), into chunks that go round-robin over
// the devices; H2D of chunk c+1, kernels of chunk c and
// D2H of chunk c-1 overlap on every device, and every chunk's tokens land at their final offset of ONE pinned
// result buffer (the "gather" of SURVEY 8(e) is a host prefix sum over per-chunk counts).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/b200bpe.h"
#include "dev_common.cuh"
#include "kernels_pretok.cuh"
#include "kernels_long.cuh"
#include "kernels_mid.cuh"
#include "kernels_pmerge.cuh"
#include "kernels_encode.cuh"
#include "kernels_special.cuh"
#include "kernels_decode.cuh"
#include "kernels_bytes.cuh"
#include "kernels_unstable.cuh"
#include "kernels_train.cuh"
#include "doc_seams.h"
#include "unicode_classes.inc"

using namespace b2bpe;

// --------------------------------------------------------------------------------------------
// error plumbing
// --------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;
static int fail(int code, const std::string &msg) { g_last_error = msg; return code; }
#define CUDA_TRY(expr)                                                                             \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return fail(B200BPE_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));        \
    } while (0)

namespace {

// pat_strs of tiktoken_ext/openai_public.py:12-14, :89, :104-114
const char *R50K_PAT = R"('(?:[sdmt]|ll|ve|re)| ?\p{L}++| ?\p{N}++| ?[^\s\p{L}\p{N}]++|\s++$|\s+(?!\S)|\s)";
const char *CL100K_PAT =
    R"('(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}++|\p{N}{1,3}+| ?[^\s\p{L}\p{N}]++[\r\n]*+|\s++$|\s*[\r\n]|\s+(?!\S)|\s)";
const char *O200K_PAT =
    R"([^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]*[\p{Ll}\p{Lm}\p{Lo}\p{M}]+(?i:'s|'t|'re|'ve|'m|'ll|'d)?|)"
    R"([^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]+[\p{Ll}\p{Lm}\p{Lo}\p{M}]*(?i:'s|'t|'re|'ve|'m|'ll|'d)?|)"
    R"(\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n/]*|\s*[\r\n]+|\s+(?!\S)|\s+)";

// the PAT_* of pat_str, else -1 (and the B200BPE_EPATTERN message)
int pattern_of(const char *pat_str) {
    if (strcmp(pat_str, R50K_PAT) == 0) return PAT_R50K;
    if (strcmp(pat_str, CL100K_PAT) == 0) return PAT_CL100K;
    if (strcmp(pat_str, O200K_PAT) == 0) return PAT_O200K;
    fail(B200BPE_EPATTERN, "unsupported pat_str: the GPU pre-tokeniser implements exactly the r50k/p50k, cl100k and "
                           "o200k patterns of tiktoken_ext/openai_public.py (there is no CPU regex fallback)");
    return -1;
}

// the calling thread's current device is restored when an ABI call returns (torch and friends keep per-thread state)
struct DeviceGuard {
    int prev = -1;
    DeviceGuard() { if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; cudaGetLastError(); } }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

template <class Tp>
struct DevBuf {
    Tp *p = nullptr; size_t cap = 0;
    cudaError_t ensure(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 8 + 256;
        cudaError_t e = cudaMalloc((void **)&p, want * sizeof(Tp));
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

struct PinnedBuf {
    void *p = nullptr; size_t cap = 0;
};

// What a pipeline run, a chunk, a device's worker or a whole call reports (the b200bpe_last_* getters).
struct CallStats {
    float ms[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};   // b200bpe_last_timings
    uint32_t launches = 0;
    uint32_t grown = 0, reruns = 0, token_passes = 0;
    uint64_t cls[N_CLS] = {}; int lane_per_piece = 0;
    uint64_t bytes_repairs = 0, unstable[5] = {}, memo[3] = {};
    uint64_t seams = 0, docs_cut = 0;    // chunks that start at a seam inside a document, documents with a seam

    // the long pieces per class and the miss memo of a run whose output the call returns
    void add_output(const Counters &c) {
        for (int i = 0; i < N_CLS; i++) cls[i] += c.n_cls[i];
        memo[0] += c.n_miss; memo[1] += c.n_owner; memo[2] += c.n_unplaced;
    }
    // everything but the timings and launches
    void add_counts(const CallStats &o) {
        grown |= o.grown; reruns += o.reruns;
        for (int i = 0; i < N_CLS; i++) cls[i] += o.cls[i];
        bytes_repairs += o.bytes_repairs;
        for (int i = 0; i < 5; i++) unstable[i] += o.unstable[i];
        for (int i = 0; i < 3; i++) memo[i] += o.memo[i];
        seams += o.seams; docs_cut += o.docs_cut;
    }
    // the next chunk of the same device: timings and launches add up
    void add(const CallStats &o) {
        for (int i = 0; i < 9; i++) ms[i] += o.ms[i];
        launches += o.launches;
        add_counts(o);
    }
    // another device's worker: each timing is the slowest device's, launches add up
    void merge(const CallStats &o) {
        for (int i = 0; i < 9; i++) ms[i] = std::max(ms[i], o.ms[i]);
        launches += o.launches;
        add_counts(o);
    }
};

long env_long(const char *name, long dflt, long lo, long hi) {
    const char *v = getenv(name);
    if (!v || !*v) return dflt;
    long x = atol(v);
    return x < lo ? lo : x > hi ? hi : x;
}

// B200BPE_CHUNK_MB: the host path's chunk size in MiB (1..2048), e.g. to place chunk seams in tests; 0 when unset
size_t env_chunk_bytes() {
    const char *v = getenv("B200BPE_CHUNK_MB");
    const long x = v ? atol(v) : 0;
    return x >= 1 && x <= 2048 ? (size_t)x << 20 : 0;
}

// Persistent helper threads of one engine: they stage pageable caller memory into pinned blocks, next to the device
// pipeline (the reference's counterpart is its rayon / thread pool).
struct TaskPool {
    std::vector<std::thread> th; std::mutex mu; std::condition_variable cv; std::deque<std::function<void()>> q; bool stop = false;
    void ensure(int n) {
        std::lock_guard<std::mutex> lk(mu);
        while ((int)th.size() < n) th.emplace_back([this] {
            for (;;) {
                std::function<void()> f;
                {
                    std::unique_lock<std::mutex> lk(mu);
                    cv.wait(lk, [this] { return stop || !q.empty(); });
                    if (q.empty()) return;
                    f = std::move(q.front()); q.pop_front();
                }
                f();
            }
        });
    }
    void push(std::function<void()> f) { { std::lock_guard<std::mutex> lk(mu); q.push_back(std::move(f)); } cv.notify_one(); }
    ~TaskPool() {
        { std::lock_guard<std::mutex> lk(mu); stop = true; }
        cv.notify_all();
        for (auto &t : th) t.join();
    }
};
struct Latch {
    std::mutex mu; std::condition_variable cv; int left;
    explicit Latch(int n) : left(n) {}
    void done() { std::lock_guard<std::mutex> lk(mu); if (--left == 0) cv.notify_all(); }
    void wait() { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [this] { return left == 0; }); }
};
// fn(lo, hi) over [0, n) in blocks, on the pool; the caller waits
void pool_for(TaskPool *pool, size_t n, size_t block, const std::function<void(size_t, size_t)> &fn) {
    const size_t nb = (n + block - 1) / block;
    if (!pool || nb <= 1) { if (n) fn(0, n); return; }
    Latch latch((int)nb);
    for (size_t b = 0; b < nb; b++) pool->push([&, b] { fn(b * block, std::min(n, (b + 1) * block)); latch.done(); });
    latch.wait();
}

}  // namespace

// One pipeline slot: a stream, its events and a grow-only workspace.  The host path keeps
// three slots in flight per device (H2D of chunk c+1, kernels of chunk c, D2H of chunk c-1).
struct Slot {
    DevBuf<uint8_t> w_text; DevBuf<unsigned long long> w_docoff, w_tokoff, w_sub_base;
    DevBuf<uint32_t> w_ptok, w_mres, w_mq_pos, w_mq_roff, w_doc_tiles, w_sub_count; DevBuf<uint8_t> w_mq_len;
    DevBuf<uint4> w_mq_key, w_mq_skey, w_mq_smeta, w_mq_rec;
    DevBuf<uint4> w_memo_key; DevBuf<uint32_t> w_memo_owner, w_mq_slot, w_mq_own, w_memo_bn;   // miss memo (MissMemo)
    DevBuf<uint32_t> w_dbits, w_pbits, w_psum, w_sfd, w_lidx, w_out, w_ltok, w_hbits, w_ibits, w_sbits, w_cbits, w_slow;
    DevBuf<unsigned long long> w_lq_start, w_lq_off; DevBuf<unsigned int> w_lq_len, w_lq_ntok, w_lq_cls, w_big_n, w_sort_hist;
    DevBuf<unsigned long long> w_big_dst, w_big_src, w_scan_part;
    DevBuf<uint32_t> w_idA, w_rkA, w_idB, w_rkB, w_aux1, w_aux2; DevBuf<uint8_t> w_flag, w_spflags;
    // bytes mode: first ill-formed byte (then unstable-piece start), tokens to drop and tail bytes per document; run 2's
    // text, document offsets and output; the spliced result (swapped with w_out / w_tokoff)
    DevBuf<uint32_t> w_vup, w_kdrop, w_btail, w_b2out, w_bout; DevBuf<uint8_t> w_btext;
    DevBuf<unsigned long long> w_b2doc, w_b2off, w_bbase, w_bpart;
    // allocated by the first bytes-mode call: the splice's scan (run 2 reuses d_ctr), the repair's counters (h_bytes pinned)
    Counters *d_bctr = nullptr; BytesCounters *d_bytes = nullptr, *h_bytes = nullptr;
    // completion search: run 1's unstable tail per document (|U|, search items; tokens to drop in w_kdrop)
    DevBuf<uint32_t> w_ulen, w_unit;
    size_t long_cap = 0;            // entries of the global merge scratch (pieces > 256 bytes), grown on ERR_LONGCAP
    size_t miss_cap = 0, mres_cap = 0;   // miss queue entries / miss result tokens, grown on ERR_MISSCAP
    size_t slow_cap = 0;            // positions left to the general pre-tokeniser rule function, grown on ERR_SLOWCAP
    Counters *d_ctr = nullptr; Counters *h_ctr = nullptr;   // h_ctr pinned
    unsigned int *d_sticky = nullptr;                       // error bits of every pipeline since the last wait
    cudaStream_t stream = nullptr;
    cudaStream_t side = nullptr;     // the group kernels (17..1024 bytes) run here, next to probe + miss on the main stream,
    cudaStream_t side2 = nullptr;    // and the scratch kernels (warp / block / cluster per piece: a few SMs each) here
    cudaStream_t up = nullptr;       // host path: uploads of the slot's NEXT chunk (ordered behind the kernels, not the download, of its last one)
    static const int N_EV = 15;       // [10] fork, [11] side start, [12] side end (join), [13] side2 end (join),
                                      // [14] bytes mode: start of the tail runs
    cudaEvent_t ev[N_EV];
    PinnedBuf stage;                // pinned staging for callers whose text is pageable memory
    bool ok = false;

    cudaError_t init() {
        cudaError_t e = cudaMalloc((void **)&d_ctr, sizeof(Counters));
        if (e == cudaSuccess) e = cudaMalloc((void **)&d_sticky, 16);
        if (e == cudaSuccess) e = cudaMemset(d_sticky, 0, 16);
        if (e == cudaSuccess) e = cudaHostAlloc((void **)&h_ctr, sizeof(Counters), cudaHostAllocPortable);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&side2, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&up, cudaStreamNonBlocking);
        for (int i = 0; i < N_EV && e == cudaSuccess; i++) e = cudaEventCreate(&ev[i]);
        ok = (e == cudaSuccess);
        return e;
    }
    void release_workspace() {
        w_text.release(); w_docoff.release(); w_tokoff.release(); w_sub_base.release();
        w_ptok.release(); w_mres.release(); w_mq_pos.release(); w_mq_roff.release(); w_doc_tiles.release(); w_sub_count.release();
        w_mq_len.release(); w_mq_rec.release(); w_mq_key.release(); w_mq_skey.release(); w_mq_smeta.release();
        w_memo_key.release(); w_memo_owner.release(); w_mq_slot.release(); w_mq_own.release(); w_memo_bn.release();
        w_dbits.release(); w_pbits.release(); w_psum.release(); w_sfd.release(); w_lidx.release(); w_out.release(); w_ltok.release();
        w_hbits.release(); w_ibits.release(); w_sbits.release(); w_cbits.release(); w_slow.release(); w_spflags.release();
        w_lq_start.release(); w_lq_off.release(); w_lq_len.release(); w_lq_ntok.release(); w_lq_cls.release(); w_big_n.release();
        w_sort_hist.release(); w_big_dst.release(); w_big_src.release(); w_scan_part.release();
        w_idA.release(); w_rkA.release(); w_idB.release(); w_rkB.release(); w_aux1.release(); w_aux2.release();
        w_flag.release();
        w_vup.release(); w_kdrop.release(); w_btail.release(); w_b2out.release(); w_bout.release(); w_btext.release();
        w_b2doc.release(); w_b2off.release(); w_bbase.release(); w_bpart.release();
        w_ulen.release(); w_unit.release();
        if (stage.p) cudaFreeHost(stage.p);
        stage.p = nullptr; stage.cap = 0;
        long_cap = miss_cap = mres_cap = slow_cap = 0;
    }
    void destroy() {
        release_workspace();
        if (d_ctr) cudaFree(d_ctr);
        if (d_bctr) cudaFree(d_bctr);
        if (d_bytes) cudaFree(d_bytes);
        if (h_bytes) cudaFreeHost(h_bytes);
        if (d_sticky) cudaFree(d_sticky);
        if (h_ctr) cudaFreeHost(h_ctr);
        if (ok) { for (int i = 0; i < N_EV; i++) cudaEventDestroy(ev[i]); }
        if (stream) cudaStreamDestroy(stream);
        if (side) cudaStreamDestroy(side);
        if (side2) cudaStreamDestroy(side2);
        if (up) cudaStreamDestroy(up);
    }
};

// Completion search work-space of one device (kernels_unstable.cuh): a device searches one chunk at a time.  The search
// items and the per-round arrays are bounded by a chunk (the round's candidate count and text); only the result (the
// distinct completions) and the deduplication table grow with what the batch returns.
struct UnstWs {
    DevBuf<uint32_t> it_lo, it_cnt, it_bytes, it_doc; DevBuf<unsigned long long> item_base, cbase, tbase, part;
    DevBuf<uint4> cinfo; DevBuf<uint32_t> o_len, s_len, out_o, out_s, nkeep, slot, keep, kc;
    DevBuf<unsigned long long> o_off, s_off, tokoff_o, tokoff_s, rcb, rtb, zeros, grp_off;
    DevBuf<uint8_t> text_o, text_s;
    DevBuf<unsigned long long> tkey; DevBuf<uint32_t> tidx, tloc;
    uint32_t tslots_min = 0;                 // grown when a table ran out of slots
    DevBuf<uint32_t> res_tok, res_doc, grp; DevBuf<unsigned long long> res_off;
    UnstCounters *d_uc = nullptr, *h_uc = nullptr;   // h_uc pinned
    Counters *d_sctr = nullptr;              // the scans' total
    void release() {                         // the grow-only buffers; the counters stay
        it_lo.release(); it_cnt.release(); it_bytes.release(); it_doc.release(); item_base.release(); cbase.release();
        tbase.release(); part.release(); cinfo.release(); o_len.release(); s_len.release(); out_o.release(); out_s.release();
        nkeep.release(); slot.release(); keep.release(); kc.release(); o_off.release(); s_off.release(); tokoff_o.release();
        tokoff_s.release(); rcb.release(); rtb.release(); zeros.release(); grp_off.release(); text_o.release(); text_s.release();
        tkey.release(); tidx.release(); tloc.release(); res_tok.release(); res_doc.release(); grp.release(); res_off.release();
    }
};

// Everything that lives on one CUDA device: the replicated tables and the pipeline slots.
struct DevCtx {
    int device = 0;
    uint8_t *arena = nullptr; size_t arena_bytes = 0;                  // all tables in one allocation
    DevTables T; UcTables uc;
    uint32_t *d_tok_boff = nullptr; uint8_t *d_tok_blob = nullptr;     // decode: id -> bytes
    uint32_t *d_tok_space = nullptr;                                   // bit per id: every byte is ' ', '\n' or '\t' (uploaded by
                                                                       // the first bytes-mode call)
    SpecialTables sp;                                                  // device copy of the special-token patterns
    uint8_t *d_sp_arena = nullptr;
    UnstTables ut;                                                     // completion search tables (the first such call)
    uint8_t *d_ut_arena = nullptr;
    UnstWs uw;                                                         // completion search work-space (one chunk at a time)
    static const int N_SLOTS = 3;     // pipeline slots per device: uploads run N_SLOTS - 2 chunks ahead of the kernels
    Slot slots[N_SLOTS];
    int n_sm = 0;                     // multiprocessors: the persistent and work-queue kernels launch a multiple of this
};

struct b200bpe_result {
    b200bpe *owner = nullptr;
    PinnedBuf tok, off;                 // pinned when produced by the engine
    std::vector<uint32_t> vtok;         // used when the result is assembled on the host (fallback special path)
    std::vector<uint64_t> voff;
    std::vector<uint64_t> vgrp;         // completions of b200bpe_encode_with_unstable_batch: per input document, its range
    bool on_host_vec = false;
    uint64_t n_tokens = 0, n_docs = 0;
};

struct PendingDeviceCall {             // the most recent b200bpe_encode_device*_async call (for b200bpe_device_wait*)
    bool active = false; int queued = 0;
    const uint8_t *d_text = nullptr; uint64_t n_bytes = 0; const unsigned long long *d_doc_off = nullptr; uint64_t n_docs = 0;
    uint32_t *d_tokens = nullptr;         // NULL: count only
    unsigned long long *d_tok_off = nullptr; unsigned long long *d_counts = nullptr;
    std::vector<uint8_t> sp_flags;        // the caller's special-token flags, copied (a re-run outlives the caller's array); empty: none
    cudaStream_t st = nullptr;
    CallStats run;                        // the launches of its enqueue; the wait adds what it collects
};

struct b200bpe {
    int pattern = 0;
    HostTables H;
    std::vector<std::string> specials; std::vector<uint32_t> special_rank;
    std::unordered_map<uint32_t, std::string> special_decoder;
    SpecialHost sp_host;                // hash table of the specials (built once), uploaded to every device
    uint32_t n_ids = 0; bool decode_on_device = true;
    std::vector<uint32_t> tok_space;    // bit per id: all-space token (bytes mode; each device gets a copy on first use)
    std::vector<DevCtx *> devs;
    uint64_t table_bytes[4] = {0, 0, 0, 0};
    // what the most recent call reported; every encode entry point resets it before its argument checks and outside
    // h->mu, hence a mutex of its own
    std::mutex stats_mu; CallStats last;
    void reset_stats() {                 // timings and launches stay those of the call before
        std::lock_guard<std::mutex> lk(stats_mu);
        CallStats z;
        memcpy(z.ms, last.ms, sizeof(z.ms)); z.launches = last.launches;
        last = z;
    }
    CallStats stats() { std::lock_guard<std::mutex> lk(stats_mu); return last; }
    void publish(const CallStats &s) { std::lock_guard<std::mutex> lk(stats_mu); last = s; }
    void publish_timings(const CallStats &s) {
        std::lock_guard<std::mutex> lk(stats_mu);
        memcpy(last.ms, s.ms, sizeof(s.ms)); last.launches = s.launches;
    }
    // a call that returns no output: what it redid and, with timings, the timings and launches of its runs
    void publish_redo(const CallStats &s, bool timings = false) {
        std::lock_guard<std::mutex> lk(stats_mu);
        last.grown = s.grown; last.reruns = s.reruns; last.token_passes = s.token_passes;
        if (timings) { memcpy(last.ms, s.ms, sizeof(s.ms)); last.launches = s.launches; }
    }
    // completion search tables on the host, built by the first b200bpe_encode_with_unstable_batch call (then uploaded to
    // every device): mergeable ids in byte order, prefix sums of their lengths, all-space bits of the mergeable tokens,
    // per-id UTF-8 facts, and the byte_pair_encode of every token its own merges do not reach
    struct {
        bool built = false;
        std::vector<uint32_t> sorted, space, ur_idx, ur_off, ur_tok; std::vector<unsigned long long> lenpre;
        std::vector<uint8_t> u8info; uint32_t max_len = 0;
    } uh;
    size_t chunk_bytes = 64u << 20; bool chunk_forced = false;
    int copy_threads = 4;
    TaskPool *pool = nullptr;        // helper threads (created with the first host-path call)
    long memo_slots = -1;            // miss memo slots per call: -1 from the batch size, 0 off (B200BPE_MISS_MEMO_SLOTS)
    bool mid_group = true;           // 17..1024-byte pieces: group-of-lanes and parallel-merge kernels (need ranks < 2^22)
    std::mutex mu;
    std::vector<PinnedBuf> pinned_pool;
    // results keep the engine alive: b200bpe_destroy with results outstanding only marks the handle dead, the last
    // b200bpe_result_free tears it down (the reference's TiktokenBuffer owns its Vec, src/py.rs:186-189)
    int live_results = 0;
    bool dead = false;
    PendingDeviceCall pending;

    PinnedBuf take_pinned(size_t bytes) {
        for (size_t i = 0; i < pinned_pool.size(); i++)
            if (pinned_pool[i].cap >= bytes && pinned_pool[i].cap <= 2 * bytes + (64u << 20)) {
                PinnedBuf b = pinned_pool[i]; pinned_pool.erase(pinned_pool.begin() + i); return b;
            }
        PinnedBuf b; size_t want = bytes + bytes / 8 + 4096;
        if (cudaHostAlloc(&b.p, want, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); b.p = nullptr; b.cap = 0; return b; }
        b.cap = want; return b;
    }
    void give_pinned(PinnedBuf b) {
        if (!b.p) return;
        if (pinned_pool.size() >= 4) {                     // keep the largest blocks
            size_t mn = 0;
            for (size_t i = 1; i < pinned_pool.size(); i++) if (pinned_pool[i].cap < pinned_pool[mn].cap) mn = i;
            if (pinned_pool[mn].cap >= b.cap) { cudaFreeHost(b.p); return; }
            cudaFreeHost(pinned_pool[mn].p); pinned_pool[mn] = b; return;
        }
        pinned_pool.push_back(b);
    }
};

extern "C" const char *b200bpe_last_error(void) { return g_last_error.c_str(); }
extern "C" const char *b200bpe_version(void) { return "b200bpe 0.2 (sm_90a)"; }
extern "C" int b200bpe_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

// --------------------------------------------------------------------------------------------
// construction
// --------------------------------------------------------------------------------------------
static void devctx_destroy(DevCtx *D) {
    if (!D) return;
    cudaSetDevice(D->device);
    for (int i = 0; i < DevCtx::N_SLOTS; i++) D->slots[i].destroy();
    if (D->arena) cudaFree(D->arena);
    if (D->d_tok_boff) cudaFree(D->d_tok_boff);
    if (D->d_tok_blob) cudaFree(D->d_tok_blob);
    if (D->d_tok_space) cudaFree(D->d_tok_space);
    if (D->d_sp_arena) cudaFree(D->d_sp_arena);
    if (D->d_ut_arena) cudaFree(D->d_ut_arena);
    D->uw.release();
    if (D->uw.d_uc) cudaFree(D->uw.d_uc);
    if (D->uw.h_uc) cudaFreeHost(D->uw.h_uc);
    if (D->uw.d_sctr) cudaFree(D->uw.d_sctr);
    delete D;
}

// the pre-tokeniser's class of every ASCII byte (its fast path), from the two-stage Unicode class tables
static void uc_ascii_table(uint8_t *ascii) {
    for (int i = 0; i < 128; i++) ascii[i] = UC_STAGE2[(uint32_t)UC_STAGE1[0] * 256 + i];
}

static int devctx_create(b200bpe *h, int device, const std::vector<uint32_t> &boff, const std::vector<uint8_t> &blob,
                         DevCtx **out) {
    DevCtx *D = new DevCtx();
    D->device = device;
    const HostTables &H = h->H;
    cudaError_t e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&D->n_sm, cudaDevAttrMultiProcessorCount, device);
    uint8_t ascii[128];
    uc_ascii_table(ascii);
    // one arena, hottest tables first
    struct Part { const void *src; size_t bytes; size_t off; };
    enum { P_NARROW, P_WIDE, P_PAIR2, P_BYTE_ID, P_PAIR, P_ASCII, P_UC1, P_UC2, P_LONG, P_BLOB, N_PARTS };
    Part parts[N_PARTS] = {{H.narrow_tab.data(), H.narrow_tab.size() * sizeof(U4), 0},
                           {H.wide_tab.data(), H.wide_tab.size() * sizeof(U4), 0}, {H.pair2.data(), 65536 * 4, 0},
                           {H.byte_id.data(), 256 * 4, 0}, {H.pair_tab.data(), H.pair_tab.size() * sizeof(U4), 0},
                           {ascii, 128, 0}, {UC_STAGE1, sizeof(UC_STAGE1), 0}, {UC_STAGE2, sizeof(UC_STAGE2), 0},
                           {H.long_tab.data(), H.long_tab.size() * sizeof(U4), 0}, {H.long_blob.data(), H.long_blob.size(), 0}};
    size_t total = 0;
    for (auto &p : parts) { p.off = total; total += (p.bytes + 255) & ~(size_t)255; }
    D->arena_bytes = total;
    if (e == cudaSuccess) e = cudaMalloc((void **)&D->arena, total);
    for (auto &p : parts) if (e == cudaSuccess && p.bytes) e = cudaMemcpy(D->arena + p.off, p.src, p.bytes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc((void **)&D->d_tok_boff, boff.size() * 4);
    if (e == cudaSuccess) e = cudaMemcpy(D->d_tok_boff, boff.data(), boff.size() * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc((void **)&D->d_tok_blob, blob.size());
    if (e == cudaSuccess) e = cudaMemcpy(D->d_tok_blob, blob.data(), blob.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = special_upload(h->sp_host, &D->d_sp_arena, &D->sp);
    for (int i = 0; i < DevCtx::N_SLOTS && e == cudaSuccess; i++) e = D->slots[i].init();
    if (e == cudaSuccess) e = cudaFuncSetAttribute(mid_thread_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MID_SMEM_BYTES);
    if (e != cudaSuccess) { std::string m = cudaGetErrorString(e); devctx_destroy(D); return fail(B200BPE_ECUDA, "device " + std::to_string(device) + " setup: " + m); }
    D->T.narrow_tab = (const U4 *)(D->arena + parts[P_NARROW].off); D->T.narrow_mask = H.narrow_mask;
    D->T.wide_tab = (const U4 *)(D->arena + parts[P_WIDE].off); D->T.wide_mask = H.wide_mask;
    D->T.pair2 = (const uint32_t *)(D->arena + parts[P_PAIR2].off);
    D->T.byte_id = (const uint32_t *)(D->arena + parts[P_BYTE_ID].off);
    D->T.pair_tab = (const U4 *)(D->arena + parts[P_PAIR].off); D->T.pair_mask = H.pair_mask;
    D->uc.ascii = D->arena + parts[P_ASCII].off;
    D->uc.stage1 = (const uint16_t *)(D->arena + parts[P_UC1].off);
    D->uc.stage2 = D->arena + parts[P_UC2].off;
    D->uc.one = 1u;
    D->T.long_tab = (const U4 *)(D->arena + parts[P_LONG].off); D->T.long_mask = H.long_mask;
    D->T.long_blob = D->arena + parts[P_BLOB].off;
    D->T.max_token_len = H.max_token_len; D->T.n_long_tokens = H.n_long_tokens;
    *out = D;
    return B200BPE_OK;
}

extern "C" int b200bpe_create_multi(const uint8_t *tok_bytes, const uint64_t *tok_off, const uint32_t *tok_rank,
                                    uint32_t n_tok, const uint8_t *sp_bytes, const uint64_t *sp_off,
                                    const uint32_t *sp_rank, uint32_t n_sp, const char *pat_str, const int *devices,
                                    int n_dev, b200bpe_t **out) {
    if (!out || !pat_str || (n_tok && (!tok_bytes || !tok_off || !tok_rank)) || !devices || n_dev < 1)
        return fail(B200BPE_EINVAL, "null argument");
    const int pattern = pattern_of(pat_str);
    if (pattern < 0) return B200BPE_EPATTERN;
    // the probe kernel tags a piece's token slot with the top two bits (kernels_encode.cuh PT_KIND), special ids included:
    // like the mergeable ranks (build_tables), every special id must stay below them
    for (uint32_t i = 0; i < n_sp; i++)
        if (sp_rank[i] >= (1u << 30)) return fail(B200BPE_EINVAL, "special token id too large (token ids must be < 2^30)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(B200BPE_ECUDA, "no CUDA device: libb200bpe has no CPU fallback");
    }
    for (int i = 0; i < n_dev; i++) {
        if (devices[i] < 0 || devices[i] >= ndev) return fail(B200BPE_EINVAL, "bad device index");
        for (int j = 0; j < i; j++) if (devices[j] == devices[i]) return fail(B200BPE_EINVAL, "duplicate device index");
    }
    DeviceGuard guard;
    b200bpe *h = new b200bpe();
    h->pattern = pattern;
    int rc = build_tables(tok_bytes, tok_off, tok_rank, n_tok, h->H);
    if (rc) { std::string m = h->H.error; delete h; return fail(rc == -3 ? B200BPE_EDUPRANK : B200BPE_EINVAL, m); }
    for (uint32_t i = 0; i < n_sp; i++) {
        std::string s((const char *)sp_bytes + sp_off[i], (size_t)(sp_off[i + 1] - sp_off[i]));
        h->specials.push_back(s); h->special_rank.push_back(sp_rank[i]);
        h->special_decoder[sp_rank[i]] = s;
    }
    special_build(h->specials, h->special_rank, h->sp_host);
    const HostTables &H = h->H;
    // decode tables: byte offsets by token id (mergeable ranks and specials).  Ids of 2^24 and above do not get a
    // dense table: with any such id the batched decode runs on the host maps (same results, KeyError included).
    uint32_t max_id = 0; bool any = false;
    for (auto &kv : H.decoder) { if (kv.first >= (1u << 24)) h->decode_on_device = false; else { max_id = std::max(max_id, kv.first); any = true; } }
    for (auto &kv : h->special_decoder) { if (kv.first >= (1u << 24)) h->decode_on_device = false; else { max_id = std::max(max_id, kv.first); any = true; } }
    h->n_ids = any ? max_id + 1 : 0;
    std::vector<uint32_t> boff((size_t)h->n_ids + 2, 0);
    std::vector<uint8_t> blob;
    std::vector<uint32_t> &space = h->tok_space;
    space.assign((size_t)h->n_ids / 32 + 2, 0);                  // token_is_all_space of lib.rs:455-465, per id
    for (uint32_t id = 0; id < h->n_ids; id++) {
        boff[id] = (uint32_t)blob.size();
        const std::string *sp = nullptr;
        auto it = H.decoder.find(id);
        if (it != H.decoder.end()) sp = &it->second;
        else { auto it2 = h->special_decoder.find(id); if (it2 != h->special_decoder.end()) sp = &it2->second; }
        if (sp) {
            blob.insert(blob.end(), sp->begin(), sp->end());
            bool all = !sp->empty();
            for (char c : *sp) all &= c == ' ' || c == '\n' || c == '\t';
            if (all) space[id >> 5] |= 1u << (id & 31);
        }
    }
    boff[h->n_ids] = (uint32_t)blob.size(); boff[h->n_ids + 1] = (uint32_t)blob.size();
    if (blob.empty()) blob.push_back(0);
    for (int i = 0; i < n_dev; i++) {
        DevCtx *D = nullptr;
        rc = devctx_create(h, devices[i], boff, blob, &D);
        if (rc) { for (auto *d : h->devs) devctx_destroy(d); delete h; return rc; }
        h->devs.push_back(D);
    }
    if (const size_t cb = env_chunk_bytes()) { h->chunk_bytes = cb; h->chunk_forced = true; }
    h->mid_group = H.max_rank < MIDG_MAX_RANK;
    h->memo_slots = env_long("B200BPE_MISS_MEMO_SLOTS", -1, 0, 1l << 24);
    h->copy_threads = (int)env_long("B200BPE_COPY_THREADS", std::max(1u, std::min(16u, std::thread::hardware_concurrency() / 4)), 1, 64);
    h->table_bytes[0] = (H.narrow_tab.size() + H.wide_tab.size()) * sizeof(U4);
    h->table_bytes[1] = H.pair_tab.size() * sizeof(U4) + 65536 * 4 + 1024;
    h->table_bytes[2] = H.long_tab.size() * sizeof(U4) + H.long_blob.size();
    h->table_bytes[3] = sizeof(UC_STAGE1) + sizeof(UC_STAGE2) + 128;
    *out = h;
    return B200BPE_OK;
}

extern "C" int b200bpe_create(const uint8_t *tok_bytes, const uint64_t *tok_off, const uint32_t *tok_rank,
                              uint32_t n_tok, const uint8_t *sp_bytes, const uint64_t *sp_off,
                              const uint32_t *sp_rank, uint32_t n_sp, const char *pat_str, int device,
                              b200bpe_t **out) {
    return b200bpe_create_multi(tok_bytes, tok_off, tok_rank, n_tok, sp_bytes, sp_off, sp_rank, n_sp, pat_str, &device, 1, out);
}

static void engine_teardown(b200bpe *h) {
    DeviceGuard guard;
    for (auto *d : h->devs) devctx_destroy(d);
    for (auto &b : h->pinned_pool) cudaFreeHost(b.p);
    delete h->pool;
    delete h;
}

extern "C" void b200bpe_destroy(b200bpe_t *h) {
    if (!h) return;
    {
        std::lock_guard<std::mutex> lk(h->mu);
        if (h->live_results > 0) { h->dead = true; return; }
    }
    engine_teardown(h);
}

extern "C" int b200bpe_n_devices(b200bpe_t *h) { return h ? (int)h->devs.size() : 0; }

// Give the grow-only work-spaces (about 25 bytes of device memory per input byte of the largest batch seen, per pipeline
// slot) and the pooled pinned result blocks back; the tables stay.  The next call re-allocates what it needs.
extern "C" int b200bpe_trim(b200bpe_t *h) {
    if (!h) return fail(B200BPE_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(h->mu);
    if (h->pending.active) return fail(B200BPE_EINVAL, "a device call is in flight: b200bpe_device_wait first");
    DeviceGuard guard;
    for (auto *D : h->devs) {
        CUDA_TRY(cudaSetDevice(D->device));
        for (int i = 0; i < DevCtx::N_SLOTS; i++) {
            CUDA_TRY(cudaStreamSynchronize(D->slots[i].stream));
            CUDA_TRY(cudaStreamSynchronize(D->slots[i].side));
            CUDA_TRY(cudaStreamSynchronize(D->slots[i].side2));
            D->slots[i].release_workspace();
        }
        D->uw.release();
    }
    for (auto &b : h->pinned_pool) cudaFreeHost(b.p);
    h->pinned_pool.clear();
    return B200BPE_OK;
}

// --------------------------------------------------------------------------------------------
// the device pipeline
// --------------------------------------------------------------------------------------------
struct PipeArgs {
    const uint8_t *d_text = nullptr; uint64_t n_bytes = 0;
    const unsigned long long *d_doc_off = nullptr; uint64_t n_docs = 0;
    uint32_t *d_out = nullptr;                   // NULL: count only (token offsets and counts, no tokens)
    unsigned long long *d_tok_off = nullptr;
    unsigned long long *d_counts = nullptr;      // optional device u64[2]: {n_tokens, n_docs} (for a count exchange)
    cudaStream_t st = nullptr;
    bool single_piece = false;                   // every document is one piece (P = D)
    bool bytes = false;                          // bytes mode: documents need not be UTF-8 (kernels_bytes.cuh)
    bool unstable = false;                       // completion search: run 1 also finds every document's unstable tail
    const uint8_t *sp_flags = nullptr;           // host: per special 1 = allowed, 2 = disallowed (NULL: no special handling)
};

static const unsigned long long MISS_CAP_MIN = 1u << 16, LONG_CAP_MIN = 1u << 20;

// exclusive scan of n u32 counts into base[0..n] (base[n] = the sum, also in ctr->total_tokens), on st: three launches,
// none when n == 0
static cudaError_t enqueue_scan(const uint32_t *cnt, uint64_t n, unsigned long long *part, unsigned long long *base,
                                Counters *ctr, cudaStream_t st) {
    if (n == 0) {
        cudaError_t e = cudaMemsetAsync(base, 0, 8, st);
        return e != cudaSuccess ? e : cudaMemsetAsync(&ctr->total_tokens, 0, sizeof(ctr->total_tokens), st);
    }
    const long long nb = (long long)((n + SCAN_ITEMS - 1) / SCAN_ITEMS);
    scan_partial_kernel<<<(unsigned)nb, 256, 0, st>>>(cnt, (long long)n, part);
    scan_top_kernel<<<1, 1024, 0, st>>>(part, nb, ctr);
    scan_final_kernel<<<(unsigned)nb, 256, 0, st>>>(cnt, (long long)n, part, base, ctr);
    return cudaSuccess;
}

// The pre-tokeniser of `pattern` over n_words words of text: the fast rules, then the positions they left undecided
// (two launches).  bytes: the haystack starts hbits may cut a document anywhere (kernels_bytes.cuh).
static void enqueue_pretok(int pattern, bool bytes, int n_sm, cudaStream_t st, const uint8_t *text, long long n_bytes,
                           const uint32_t *hbits, const UcTables &uc, uint32_t *pbits, uint32_t *psum, long long n_words,
                           const uint32_t *ibits, uint32_t *slow, uint32_t scap, Counters *ctr) {
    const unsigned grid = (unsigned)((n_words + 255) / 256);
    auto launch = [&](auto pat) {
        constexpr int P = decltype(pat)::value;
        if (bytes) pretok_kernel<P, true><<<grid, 256, 0, st>>>(text, n_bytes, hbits, uc, pbits, psum, n_words, ibits, slow, scap, ctr);
        else pretok_kernel<P><<<grid, 256, 0, st>>>(text, n_bytes, hbits, uc, pbits, psum, n_words, ibits, slow, scap, ctr);
        pretok_slow_kernel<P><<<n_sm * 8, 256, 0, st>>>(text, n_bytes, hbits, uc, pbits, psum, slow, scap, ctr);
    };
    if (pattern == PAT_R50K) launch(std::integral_constant<int, PAT_R50K>());
    else if (pattern == PAT_CL100K) launch(std::integral_constant<int, PAT_CL100K>());
    else launch(std::integral_constant<int, PAT_O200K>());
}

// Enqueue the whole pipeline on args.st; run.launches = its kernel launches.  All pointers are device pointers on
// D->device; d_text must be 16-byte aligned and readable up to n_bytes + 16.  No host synchronisation.
static int enqueue_pipeline(b200bpe *h, DevCtx *D, Slot &S, const PipeArgs &a, CallStats &run) {
    const uint64_t n_bytes = a.n_bytes, n_docs = a.n_docs;
    cudaStream_t st = a.st;
    if (n_bytes >= (1ull << 32) - 4096) return fail(B200BPE_EINVAL, "batch too large for one call (>= 4 GiB)");
    if (n_docs >= 0xFFFFFFFEull) return fail(B200BPE_EINVAL, "too many documents in one call");
    const bool count_only = a.d_out == nullptr;
    if (count_only && (a.bytes || a.unstable))
        return fail(B200BPE_EINVAL, "bytes mode and the completion search need the tokens: no count-only call");
    const long long n_words = (long long)((n_bytes + 1 + 31) / 32);
    const long long n_tiles = (n_words + 31) / 32;                  // 1 KiB sub-tiles
    const size_t pb_words = (size_t)n_tiles * 32 + STAGE_PW + 8;    // the probe stages 36 words per sub-tile
    CUDA_TRY(S.w_dbits.ensure((size_t)n_words + 8));
    CUDA_TRY(S.w_pbits.ensure(pb_words));
    CUDA_TRY(S.w_psum.ensure((size_t)(n_words >> 5) + 4));
    CUDA_TRY(S.w_sfd.ensure((size_t)n_words + 4));
    CUDA_TRY(S.w_sub_base.ensure((size_t)n_tiles + 2));
    CUDA_TRY(S.w_scan_part.ensure((size_t)(n_tiles / SCAN_ITEMS) + 4));
    CUDA_TRY(S.w_sub_count.ensure((size_t)n_tiles + 2));
    CUDA_TRY(S.w_ptok.ensure((size_t)n_tiles * SUB_BYTES + 64));
    {   // miss queue: sized from experience (one miss per 8 bytes, two result tokens per 4 bytes), grown on ERR_MISSCAP
        const size_t want_q = std::max<size_t>((size_t)(n_bytes / 8) + 4096, MISS_CAP_MIN);
        const size_t want_r = std::max<size_t>((size_t)(n_bytes / 2) + 4096, MISS_CAP_MIN);
        if (S.miss_cap < want_q) S.miss_cap = want_q;
        if (S.mres_cap < want_r) S.mres_cap = want_r;
        const size_t mcap = S.miss_cap;
        CUDA_TRY(S.w_mq_pos.ensure(mcap)); CUDA_TRY(S.w_mq_roff.ensure(mcap)); CUDA_TRY(S.w_mq_rec.ensure(mcap));
        CUDA_TRY(S.w_mq_len.ensure(mcap));
        CUDA_TRY(S.w_mq_key.ensure(mcap)); CUDA_TRY(S.w_mq_skey.ensure(mcap)); CUDA_TRY(S.w_mq_smeta.ensure(mcap));
        CUDA_TRY(S.w_mres.ensure(S.mres_cap + 64));
        CUDA_TRY(S.w_sort_hist.ensure((size_t)D->n_sm * SORT_BLOCKS_PER_SM * 17 + 32));
        CUDA_TRY(S.w_mq_slot.ensure(mcap)); CUDA_TRY(S.w_mq_own.ensure(mcap));
        CUDA_TRY(S.w_memo_bn.ensure((size_t)D->n_sm * SORT_BLOCKS_PER_SM * 2 + 4));
    }
    // miss memo: one slot per 128 bytes of text (a 16-byte key and a u32 owner), from 2^12 to 2^21 slots
    uint32_t memo_slots = 0;
    if (h->memo_slots) {
        const uint64_t want = h->memo_slots > 0 ? (uint64_t)h->memo_slots
                                                : std::min<uint64_t>(std::max<uint64_t>(n_bytes / 128, 1u << 12), 1u << 21);
        memo_slots = 1;
        while (memo_slots < want) memo_slots <<= 1;
        CUDA_TRY(S.w_memo_key.ensure(memo_slots)); CUDA_TRY(S.w_memo_owner.ensure(memo_slots));
    }
    {   // undecided pre-tokeniser positions: under 2 % on the worst corpus seen; sized for 12 %, grown on ERR_SLOWCAP
        const size_t want = std::max<size_t>((size_t)(n_bytes / 8) + 4096, MISS_CAP_MIN);
        if (S.slow_cap < want) S.slow_cap = want;
        CUDA_TRY(S.w_slow.ensure(S.slow_cap));
    }
    CUDA_TRY(S.w_lidx.ensure((size_t)(n_bytes >> 4) + 4));
    CUDA_TRY(S.w_ltok.ensure((size_t)n_bytes + 4));
    const size_t qcap = (size_t)(n_bytes / (SHORT_MAX + 1)) + 4;
    CUDA_TRY(S.w_lq_start.ensure(qcap)); CUDA_TRY(S.w_lq_off.ensure(qcap));
    CUDA_TRY(S.w_lq_len.ensure(qcap)); CUDA_TRY(S.w_lq_ntok.ensure(qcap));
    size_t cls_cap[N_CLS], cls_total = 0;                          // per-class index lists, back to back
    {
        const size_t min_len[N_CLS] = {SHORT_MAX + 1, 33, 65, 129, 257, GROUP_MAX + 1, BLOCK_MIN + 1, CLUSTER_MIN + 1};
        for (int c = 0; c < N_CLS; c++) { cls_cap[c] = (size_t)(n_bytes / min_len[c]) + 4; cls_total += cls_cap[c]; }
    }
    CUDA_TRY(S.w_lq_cls.ensure(cls_total));
    CUDA_TRY(S.w_big_n.ensure((size_t)(n_bytes / 4097) + 4));
    CUDA_TRY(S.w_big_dst.ensure((size_t)(n_bytes / 4097) + 4)); CUDA_TRY(S.w_big_src.ensure((size_t)(n_bytes / 4097) + 4));
    {   // global merge scratch of the pieces > 256 bytes: sized from experience, grown on ERR_LONGCAP
        const size_t want = std::max<size_t>((size_t)(n_bytes / 8) + 4096, LONG_CAP_MIN);
        if (S.long_cap < want) S.long_cap = want;
        const size_t lc = S.long_cap + 4;
        CUDA_TRY(S.w_idA.ensure(lc)); CUDA_TRY(S.w_rkA.ensure(lc)); CUDA_TRY(S.w_idB.ensure(lc)); CUDA_TRY(S.w_rkB.ensure(lc));
        CUDA_TRY(S.w_aux1.ensure(lc)); CUDA_TRY(S.w_aux2.ensure(lc)); CUDA_TRY(S.w_flag.ensure(lc));
    }
    LongQ q;
    q.start = S.w_lq_start.p; q.len = S.w_lq_len.p; q.off = S.w_lq_off.p; q.ntok = S.w_lq_ntok.p; q.scratch_cap = S.long_cap;
    q.sub_count = S.w_sub_count.p;
    { size_t o = 0; for (int c = 0; c < N_CLS; c++) { q.cls[c] = S.w_lq_cls.p + o; o += cls_cap[c]; } }
    // documents are sparse when fewer than one sub-tile in four can hold a document start: the gather then takes the
    // doc-start sub-tiles from a list instead of giving every sub-tile the shared memory their bookkeeping needs
    const bool sparse_docs = (n_docs + 1) * 4 < (uint64_t)n_tiles;
    if (sparse_docs) CUDA_TRY(S.w_doc_tiles.ensure((size_t)n_docs + 8));
    uint32_t launches = 0;

    CUDA_TRY(cudaEventRecord(S.ev[0], st));
    CUDA_TRY(cudaMemsetAsync(S.d_ctr, 0, sizeof(Counters), st));
    CUDA_TRY(cudaMemsetAsync(S.w_dbits.p, 0, ((size_t)n_words + 8) * 4, st));
    CUDA_TRY(cudaMemsetAsync(S.w_sfd.p, 0xFF, ((size_t)n_words + 4) * 4, st));
    CUDA_TRY(cudaMemsetAsync(S.w_sub_count.p, 0, ((size_t)n_tiles + 2) * 4, st));
    CUDA_TRY(cudaMemsetAsync(S.w_pbits.p + n_words, 0, (pb_words - (size_t)n_words) * 4, st));
    {
        unsigned long long nd1 = n_docs + 1;
        mark_docs_kernel<<<(unsigned)((nd1 + 255) / 256), 256, 0, st>>>(a.d_doc_off, n_docs, n_bytes, S.w_dbits.p, S.w_sfd.p,
                                                                       sparse_docs ? S.w_doc_tiles.p : nullptr, S.d_ctr);
        launches++;
    }
    // ---- special tokens (CoreBPE::encode, lib.rs:375-442; disallowed check, core.py:120-124) ------------------
    const uint32_t *hbits = S.w_dbits.p;         // haystack starts seen by the pre-tokeniser (= documents unless cut)
    const uint32_t *ibits = nullptr, *sbits = nullptr;
    if (a.sp_flags && !h->specials.empty() && !a.single_piece) {
        const size_t nsp = h->specials.size();
        CUDA_TRY(S.w_spflags.ensure(nsp + 16));
        CUDA_TRY(S.w_hbits.ensure((size_t)n_words + 8)); CUDA_TRY(S.w_ibits.ensure((size_t)n_words + 8));
        CUDA_TRY(S.w_sbits.ensure((size_t)n_words + 8)); CUDA_TRY(S.w_cbits.ensure((size_t)n_words + 8));
        CUDA_TRY(cudaMemcpyAsync(S.w_spflags.p, a.sp_flags, nsp, cudaMemcpyHostToDevice, st));   // tiny, from the caller's array
        CUDA_TRY(cudaMemsetAsync(S.w_ibits.p, 0, ((size_t)n_words + 8) * 4, st));
        CUDA_TRY(cudaMemsetAsync(S.w_cbits.p + n_words, 0, 8 * 4, st));
        const unsigned grid = (unsigned)((n_words + 255) / 256);
        special_mark_kernel<<<grid, 256, 0, st>>>(a.d_text, (long long)n_bytes, S.w_dbits.p, D->sp, S.w_spflags.p, S.w_cbits.p, n_words, S.d_ctr);
        CUDA_TRY(cudaMemcpyAsync(S.w_hbits.p, S.w_dbits.p, ((size_t)n_words + 8) * 4, cudaMemcpyDeviceToDevice, st));
        special_resolve_kernel<<<grid, 256, 0, st>>>(a.d_text, (long long)n_bytes, S.w_dbits.p, D->sp, S.w_spflags.p, S.w_cbits.p,
                                                     S.w_hbits.p, S.w_ibits.p, S.w_sbits.p, S.w_ltok.p, n_words, S.d_ctr);
        launches += 2;
        hbits = S.w_hbits.p; ibits = S.w_ibits.p; sbits = S.w_sbits.p;
    } else if (a.bytes) {
        // ordinary semantics, so the special scan does not run and the cut owns its buffers: a document whose first
        // ill-formed byte is v gets a haystack start at v and one placeholder slot for (v, end), like an accepted special
        if (!D->d_tok_space) {
            CUDA_TRY(cudaMalloc((void **)&D->d_tok_space, h->tok_space.size() * 4));
            CUDA_TRY(cudaMemcpy(D->d_tok_space, h->tok_space.data(), h->tok_space.size() * 4, cudaMemcpyHostToDevice));
        }
        if (!S.d_bytes) CUDA_TRY(cudaMalloc((void **)&S.d_bytes, sizeof(BytesCounters)));
        if (!S.h_bytes) CUDA_TRY(cudaHostAlloc((void **)&S.h_bytes, sizeof(BytesCounters), cudaHostAllocPortable));
        CUDA_TRY(cudaMemsetAsync(S.d_bytes, 0, sizeof(BytesCounters), st));
        CUDA_TRY(S.w_hbits.ensure((size_t)n_words + 8)); CUDA_TRY(S.w_ibits.ensure((size_t)n_words + 8));
        CUDA_TRY(S.w_sbits.ensure((size_t)n_words + 8)); CUDA_TRY(S.w_vup.ensure((size_t)n_docs + 2));
        CUDA_TRY(cudaMemsetAsync(S.w_ibits.p, 0, ((size_t)n_words + 8) * 4, st));
        CUDA_TRY(cudaMemsetAsync(S.w_sbits.p, 0, ((size_t)n_words + 8) * 4, st));
        CUDA_TRY(cudaMemsetAsync(S.w_vup.p, 0xFF, ((size_t)n_docs + 2) * 4, st));
        utf8_check_kernel<<<(unsigned)((n_words + 255) / 256), 256, 0, st>>>(a.d_text, (long long)n_bytes, S.w_dbits.p, S.w_sfd.p,
                                                                            a.d_doc_off, n_docs, n_words, S.w_vup.p);
        CUDA_TRY(cudaMemcpyAsync(S.w_hbits.p, S.w_dbits.p, ((size_t)n_words + 8) * 4, cudaMemcpyDeviceToDevice, st));
        if (n_docs) bytes_cut_kernel<<<(unsigned)((n_docs * 32 + 255) / 256), 256, 0, st>>>(a.d_doc_off, n_docs, S.w_vup.p, S.w_hbits.p,
                                                                                          S.w_ibits.p, S.w_sbits.p, S.w_ltok.p);
        launches += 2;
        hbits = S.w_hbits.p; ibits = S.w_ibits.p; sbits = S.w_sbits.p;
    }
    CUDA_TRY(cudaEventRecord(S.ev[1], st));
    {
        unsigned grid = (unsigned)((n_words + 255) / 256);
        if (a.single_piece) single_piece_bits_kernel<<<grid, 256, 0, st>>>(S.w_pbits.p, S.w_psum.p, S.w_dbits.p, n_words);
        else {
            enqueue_pretok(h->pattern, a.bytes, D->n_sm, st, a.d_text, (long long)n_bytes, hbits, D->uc, S.w_pbits.p, S.w_psum.p,
                           n_words, ibits, S.w_slow.p, (uint32_t)std::min<size_t>(S.slow_cap, 0xFFFFFFF0u), S.d_ctr);
            launches++;
        }
        launches++;
    }
    CUDA_TRY(cudaEventRecord(S.ev[2], st));
    {
        unsigned grid = (unsigned)((n_words + 255) / 256);
        find_long_kernel<<<grid, 256, 0, st>>>(S.w_pbits.p, S.w_psum.p, (long long)n_bytes, n_words, q, S.w_lidx.p, sbits, S.d_ctr);
        launches++;
        // The long-piece kernels only depend on find_long and nothing before the scan depends on them: they run on a
        // side stream next to probe + miss sort + miss (few SMs are busy with a giant piece, the rest probe).
        cudaStream_t ls = S.side, ls2 = S.side2;
        CUDA_TRY(cudaEventRecord(S.ev[10], st));
        CUDA_TRY(cudaStreamWaitEvent(ls, S.ev[10], 0));
        CUDA_TRY(cudaStreamWaitEvent(ls2, S.ev[10], 0));
        CUDA_TRY(cudaEventRecord(S.ev[11], ls));
        LongScratch LS{S.w_idA.p, S.w_rkA.p, S.w_idB.p, S.w_rkB.p, S.w_aux1.p, S.w_aux2.p, S.w_flag.p};
        if (h->mid_group) {      // 129..1024 bytes: segmented parallel merge (rounds, not merges, are sequential); shorter: a group of lanes per piece
            pmerge_kernel<256, 3><<<D->n_sm * 10, PM_WARPS * 32, 0, ls>>>(a.d_text, D->T, q, S.w_ltok.p, S.d_ctr);
            pmerge_long_kernel<<<D->n_sm * 4, PM_WARPS_L * 32, 0, ls>>>(a.d_text, D->T, q, S.w_ltok.p, S.d_ctr);
            mid_group32_kernel<<<D->n_sm * 4, MIDG_WARPS * 32, 0, ls>>>(a.d_text, D->T, q, S.w_ltok.p, S.d_ctr, 2);
            mid_group16_kernel<<<D->n_sm * 9, MIDG_WARPS * 32, 0, ls>>>(a.d_text, D->T, q, S.w_ltok.p, S.d_ctr, 1);
        } else {                 // ranks of 2^22 and above: one piece per lane (72 KiB of columns per block) / warp per piece
            mid_thread_kernel<<<D->n_sm * 3, MID_WARPS * 32, MID_SMEM_BYTES, ls>>>(a.d_text, D->T, q, S.w_ltok.p, S.d_ctr);
            long_piece_kernel<<<D->n_sm * 8, LONG_WARPS * 32, 0, ls>>>(a.d_text, D->T, q, LS, S.w_ltok.p, S.d_ctr, CLS_G1024);
        }
        long_piece_kernel<<<D->n_sm * 8, LONG_WARPS * 32, 0, ls2>>>(a.d_text, D->T, q, LS, S.w_ltok.p, S.d_ctr, CLS_WARP);
        giant_piece_kernel<<<D->n_sm, GIANT_THREADS, 0, ls2>>>(a.d_text, D->T, q, LS, S.w_ltok.p, S.d_ctr);
        cluster_piece_kernel<<<(D->n_sm / CLUSTER_CTAS) * CLUSTER_CTAS, GIANT_THREADS, 0, ls2>>>(a.d_text, D->T, q, LS, S.w_ltok.p, S.d_ctr);
        CUDA_TRY(cudaEventRecord(S.ev[13], ls2));
        CUDA_TRY(cudaEventRecord(S.ev[12], ls));
        launches += 5;
    }
    CUDA_TRY(cudaEventRecord(S.ev[3], st));
    {
        TileParams p;
        p.text = a.d_text; p.n_bytes = (long long)n_bytes; p.n_words = n_words; p.n_sub = n_tiles;
        p.pbits = S.w_pbits.p; p.dbits = S.w_dbits.p; p.span_first_doc = S.w_sfd.p;
        p.doc_off = a.d_doc_off; p.n_docs = n_docs; p.q = q; p.lidx = S.w_lidx.p; p.ltok = S.w_ltok.p;
        p.ptok = S.w_ptok.p; p.mres = S.w_mres.p; p.sbits = sbits;
        p.mq.key = S.w_mq_key.p; p.mq.pos = S.w_mq_pos.p; p.mq.roff = S.w_mq_roff.p; p.mq.len = S.w_mq_len.p; p.mq.rec = S.w_mq_rec.p;
        p.doc_tiles = S.w_doc_tiles.p;
        p.mq.skey = S.w_mq_skey.p; p.mq.smeta = S.w_mq_smeta.p; p.mq.cap = (uint32_t)std::min<size_t>(S.miss_cap, 0xFFFFFFF0u);
        p.mq.mres_cap = S.mres_cap;
        p.sub_count = S.w_sub_count.p; p.sub_base = S.w_sub_base.p;
        p.out = a.d_out; p.tok_off = a.d_tok_off; p.ctr = S.d_ctr;
        p.big_dst = S.w_big_dst.p; p.big_src = S.w_big_src.p; p.big_n = S.w_big_n.p;
        MissMemo memo;
        memo.key = S.w_memo_key.p; memo.owner = S.w_memo_owner.p; memo.slot = S.w_mq_slot.p; memo.own = S.w_mq_own.p;
        memo.block_n = S.w_memo_bn.p; memo.mask = memo_slots ? memo_slots - 1 : 0; memo.on = memo_slots ? 1u : 0u;
        memo.limit = std::max<uint32_t>(1u, memo_slots / 2 / (uint32_t)(D->n_sm * SORT_BLOCKS_PER_SM));   // per dedup block
        const long long want_blocks = (n_tiles + ENC_WARPS - 1) / ENC_WARPS;
        const unsigned probe_grid = (unsigned)std::min<long long>(want_blocks, (long long)D->n_sm * PROBE_BLOCKS_PER_SM);
        probe_kernel<<<probe_grid, ENC_WARPS * 32, 0, st>>>(p, D->T);
        CUDA_TRY(cudaEventRecord(S.ev[8], st));
        const int sort_blocks = D->n_sm * SORT_BLOCKS_PER_SM;
        if (memo_slots) CUDA_TRY(cudaMemsetAsync(S.w_memo_key.p, 0, (size_t)memo_slots * sizeof(uint4), st));
        miss_dedup_kernel<<<sort_blocks, SORT_THREADS, 0, st>>>(p, memo, S.w_sort_hist.p);
        miss_base_kernel<<<1, 17 * 32, 0, st>>>(S.w_sort_hist.p, sort_blocks);
        miss_scatter_kernel<<<sort_blocks, SORT_THREADS, 0, st>>>(p, memo, S.w_sort_hist.p);
        miss_kernel<<<D->n_sm * 16, MISS_WARPS * 32, 0, st>>>(p, D->T);
        if (memo_slots) miss_fanout_kernel<<<sort_blocks, SORT_THREADS, 0, st>>>(p, memo);
        CUDA_TRY(cudaEventRecord(S.ev[7], st));
        CUDA_TRY(cudaStreamWaitEvent(st, S.ev[12], 0));          // join: the long pieces' tokens and counts are needed from here on
        CUDA_TRY(cudaStreamWaitEvent(st, S.ev[13], 0));
        CUDA_TRY(enqueue_scan(S.w_sub_count.p, (uint64_t)n_tiles, S.w_scan_part.p, S.w_sub_base.p, S.d_ctr, st));
        const unsigned gather_grid = (unsigned)((n_tiles + GATHER_WARPS - 1) / GATHER_WARPS);
        const unsigned doc_grid = (unsigned)((n_docs + 1 + GATHER_WARPS - 1) / GATHER_WARPS);
        if (count_only) {            // only the sub-tiles that hold a document start, no token stores
            if (sparse_docs) gather_kernel<1, false><<<doc_grid, GATHER_WARPS * 32, 0, st>>>(p);
            else gather_kernel<2, false><<<gather_grid, GATHER_WARPS * 32, 0, st>>>(p);
        } else {
            if (sparse_docs) {
                gather_kernel<0><<<gather_grid, GATHER_WARPS * 32, 0, st>>>(p);
                gather_kernel<1><<<doc_grid, GATHER_WARPS * 32, 0, st>>>(p);
            } else gather_kernel<2><<<gather_grid, GATHER_WARPS * 32, 0, st>>>(p);
            big_copy_kernel<<<D->n_sm * 2, 256, 0, st>>>(p);
        }
        if (a.bytes && n_docs) {     // the tokens and offsets are final: where each damaged document's unstable piece starts
            CUDA_TRY(S.w_kdrop.ensure((size_t)n_docs + 2)); CUDA_TRY(S.w_btail.ensure((size_t)n_docs + 2));
            bytes_repair_kernel<<<(unsigned)((n_docs * 32 + 255) / 256), 256, 0, st>>>(a.d_doc_off, n_docs, S.w_vup.p, S.w_pbits.p, a.d_out,
                                                                                      a.d_tok_off, D->d_tok_boff, D->d_tok_space, h->n_ids,
                                                                                      S.w_kdrop.p, S.w_btail.p, S.d_bytes, S.d_ctr);
            launches++;
        }
        if (a.unstable && n_docs) {  // the tokens and offsets are final: L, |U| and the search items of every document
            CUDA_TRY(S.w_kdrop.ensure((size_t)n_docs + 2)); CUDA_TRY(S.w_ulen.ensure((size_t)n_docs + 2));
            CUDA_TRY(S.w_unit.ensure((size_t)n_docs + 2));
            unstable_walk_kernel<<<(unsigned)((n_docs * 32 + 255) / 256), 256, 0, st>>>(a.d_doc_off, n_docs, S.w_pbits.p, sbits, a.d_out,
                                                                                       a.d_tok_off, D->d_tok_boff, D->ut.space, h->n_ids,
                                                                                       D->ut.max_len, S.w_kdrop.p, S.w_ulen.p,
                                                                                       S.w_unit.p, S.d_ctr);
            launches++;
        }
        finalize_kernel<<<1, 32, 0, st>>>(S.d_ctr, S.d_sticky, a.d_counts, n_docs);
        launches += (count_only ? 10 : sparse_docs ? 12 : 11) + (memo_slots ? 1 : 0);
    }
    CUDA_TRY(cudaEventRecord(S.ev[4], st));
    if (a.bytes) CUDA_TRY(cudaMemcpyAsync(S.h_bytes, S.d_bytes, sizeof(BytesCounters), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(S.h_ctr, S.d_ctr, sizeof(Counters), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaEventRecord(S.ev[9], st));
    run.launches = launches;
    return B200BPE_OK;
}

static const int B200BPE_RETRY = 1;      // internal: capacities were grown, run the pipeline again

// Wait for an enqueued pipeline, collect stage timings (into run.ms) and device-side flags.  Returns B200BPE_RETRY
// when a work-space that is sized from experience was too small for this batch (it has been grown to the exact need);
// the B200BPE_GREW_* bits of the work-spaces that grew are then ORed into run.grown.
static int collect_pipeline(Slot &S, CallStats &run, int *special_idx, uint64_t *special_pos) {
    CUDA_TRY(cudaEventSynchronize(S.ev[9]));
    CUDA_TRY(cudaGetLastError());
    cudaEventElapsedTime(&run.ms[0], S.ev[0], S.ev[1]);
    cudaEventElapsedTime(&run.ms[1], S.ev[1], S.ev[2]);
    cudaEventElapsedTime(&run.ms[2], S.ev[11], S.ev[12]);     // long-piece kernels (side stream, overlapped with [3])
    cudaEventElapsedTime(&run.ms[3], S.ev[3], S.ev[7]);
    cudaEventElapsedTime(&run.ms[7], S.ev[7], S.ev[4]);
    cudaEventElapsedTime(&run.ms[8], S.ev[3], S.ev[8]);
    cudaEventElapsedTime(&run.ms[4], S.ev[0], S.ev[4]);
    const Counters &c = *S.h_ctr;
    if (c.err & ERR_DOCOFF)
        return fail(B200BPE_EINVAL, "document offsets must start at 0, be non-decreasing and end at n_bytes");
    if (c.err & ERR_SPECIAL) {
        const unsigned long long packed = ~c.special_pos;       // the scan keeps max(~(pos << 16 | index)) = the leftmost match
        if (special_idx) *special_idx = (int)(packed & 0xFFFFu);
        if (special_pos) *special_pos = packed >> 16;
        return fail(B200BPE_ESPECIAL, "text contains a disallowed special token");
    }
    if (c.err & (ERR_LONGCAP | ERR_MISSCAP | ERR_SLOWCAP)) {
        if (c.err & ERR_SLOWCAP) S.slow_cap = (size_t)c.n_slow + (size_t)(c.n_slow / 8) + 4096;
        if (c.err & ERR_LONGCAP) S.long_cap = (size_t)c.long_bytes + (size_t)(c.long_bytes / 8) + 4096;
        if (c.err & ERR_MISSCAP) {
            S.miss_cap = std::max(S.miss_cap, (size_t)c.n_miss + (size_t)(c.n_miss / 8) + 4096);
            S.mres_cap = std::max(S.mres_cap, (size_t)c.miss_bytes + (size_t)(c.miss_bytes / 8) + 4096);
        }
        run.grown |= ((c.err & ERR_MISSCAP) ? B200BPE_GREW_MISS : 0u) | ((c.err & ERR_SLOWCAP) ? B200BPE_GREW_SLOW : 0u) |
                     ((c.err & ERR_LONGCAP) ? B200BPE_GREW_LONG : 0u);
        return B200BPE_RETRY;
    }
    if (c.err & ERR_INTERNAL) return fail(B200BPE_ECUDA, "internal error: a merge kernel did not converge");
    if (c.err & ERR_NOBYTE)
        return fail(B200BPE_ENOBYTE, "a piece needs a single-byte token that mergeable_ranks does not contain");
    return B200BPE_OK;
}

// Collect the run enqueued on S; while a work-space was too small (it has been grown), enqueue() the same run again and
// collect it, at most four more times.  run: the timings and launches of the last run, the re-runs, the work-spaces
// grown and, on success, the long pieces per class and miss memo counters of the last run.
static int collect_regrow(Slot &S, CallStats &run, int *special_idx, uint64_t *special_pos, const std::function<int()> &enqueue) {
    int rc = collect_pipeline(S, run, special_idx, special_pos);
    for (int attempt = 0; rc == B200BPE_RETRY && attempt < 4; attempt++) {
        rc = enqueue();
        if (!rc) { run.reruns++; rc = collect_pipeline(S, run, special_idx, special_pos); }
    }
    if (rc == B200BPE_RETRY) return fail(B200BPE_ECUDA, "work-space sizing did not converge");
    if (!rc) run.add_output(*S.h_ctr);
    return rc;
}

static bool any_flag(const b200bpe *h, const uint8_t *flags) {
    if (flags) for (size_t i = 0; i < h->specials.size(); i++) if (flags[i]) return true;
    return false;
}

static int device_enqueue_locked(b200bpe *h, const PendingDeviceCall &c, CallStats &run) {
    DevCtx *D = h->devs[0];
    Slot &S = D->slots[0];
    cudaStream_t st = c.st ? c.st : S.stream;
    const uint8_t *txt = c.d_text;
    if (((uintptr_t)c.d_text & 15u) != 0) {                       // TMA staging and vector loads need 16-byte alignment
        CUDA_TRY(S.w_text.ensure((size_t)c.n_bytes + 64));
        CUDA_TRY(cudaMemcpyAsync(S.w_text.p, c.d_text, c.n_bytes, cudaMemcpyDeviceToDevice, st));
        txt = S.w_text.p;
    }
    PipeArgs a;
    a.d_text = txt; a.n_bytes = c.n_bytes; a.d_doc_off = c.d_doc_off; a.n_docs = c.n_docs; a.d_out = c.d_tokens;
    a.d_tok_off = c.d_tok_off; a.d_counts = c.d_counts; a.st = st;
    if (!c.sp_flags.empty()) a.sp_flags = c.sp_flags.data();
    int rc = enqueue_pipeline(h, D, S, a, run);
    if (rc || !a.sp_flags) return rc;
    special_sticky_kernel<<<1, 32, 0, st>>>(S.d_ctr, S.d_sticky);
    run.launches++;
    return B200BPE_OK;
}

extern "C" int b200bpe_encode_device_special_async(b200bpe_t *h, const uint8_t *d_text, uint64_t n_bytes,
                                                   const uint64_t *d_doc_off, uint64_t n_docs, const uint8_t *flags,
                                                   uint32_t *d_tokens, uint64_t *d_tok_off, uint64_t *d_counts, void *stream) {
    if (h) h->reset_stats();
    if (!h || !d_doc_off || !d_tok_off || (n_bytes && !d_text)) return fail(B200BPE_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(h->mu);
    DeviceGuard guard;
    CUDA_TRY(cudaSetDevice(h->devs[0]->device));
    PendingDeviceCall c;
    c.active = true; c.queued = h->pending.active ? h->pending.queued + 1 : 1;
    c.d_text = d_text; c.n_bytes = n_bytes; c.d_doc_off = (const unsigned long long *)d_doc_off; c.n_docs = n_docs;
    c.d_tokens = d_tokens; c.d_tok_off = (unsigned long long *)d_tok_off; c.d_counts = (unsigned long long *)d_counts;
    c.st = (cudaStream_t)stream;
    if (any_flag(h, flags)) c.sp_flags.assign(flags, flags + h->specials.size());
    int rc = device_enqueue_locked(h, c, c.run);
    if (rc) return rc;
    h->pending = std::move(c);
    return B200BPE_OK;
}

extern "C" int b200bpe_encode_device_async(b200bpe_t *h, const uint8_t *d_text, uint64_t n_bytes, const uint64_t *d_doc_off,
                                           uint64_t n_docs, uint32_t *d_tokens, uint64_t *d_tok_off, uint64_t *d_counts,
                                           void *stream) {
    if (!d_tokens) {
        if (h) h->reset_stats();
        return fail(B200BPE_EINVAL, "null argument");
    }
    return b200bpe_encode_device_special_async(h, d_text, n_bytes, d_doc_off, n_docs, nullptr, d_tokens, d_tok_off, d_counts,
                                               stream);
}

extern "C" int b200bpe_device_wait_special(b200bpe_t *h, uint64_t *n_tokens, int32_t *special_index) {
    if (!h) return fail(B200BPE_EINVAL, "null handle");
    h->reset_stats();
    std::lock_guard<std::mutex> lk(h->mu);
    if (!h->pending.active) return fail(B200BPE_EINVAL, "no device call in flight");
    DeviceGuard guard;
    DevCtx *D = h->devs[0];
    CUDA_TRY(cudaSetDevice(D->device));
    Slot &S = D->slots[0];
    PendingDeviceCall c = h->pending;
    h->pending.active = false;
    cudaStream_t st = c.st ? c.st : S.stream;
    CallStats &run = c.run;               // grown: only what this wait grows (an earlier call of a queued series leaves sticky bits)
    run.token_passes = 1;
    int sidx = -1;
    const int rc = collect_regrow(S, run, &sidx, nullptr, [&] { return device_enqueue_locked(h, c, run); });
    h->publish_redo(run, true);           // timings (no copies: [5] = [6] = 0) and launches even when the wait fails
    // error bits of the earlier calls of a queued series (the counters only describe the last one)
    unsigned int sticky[2] = {0, 0};      // error bits, 1 + the first disallowed special (special_sticky_kernel)
    CUDA_TRY(cudaMemcpyAsync(sticky, S.d_sticky, sizeof(sticky), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemsetAsync(S.d_sticky, 0, sizeof(sticky), st));
    CUDA_TRY(cudaStreamSynchronize(st));
    // a disallowed special: the leftmost one of the earliest call of a queued series that has one.  sticky[1], not the
    // ERR_SPECIAL bit of sticky[0]: only device calls with flags set it, while finalize_kernel also ORs the error bits of
    // host-path pipelines on this slot into sticky[0] (a host call that failed on a disallowed special leaves it there)
    if (rc == B200BPE_ESPECIAL || (c.queued > 1 && sticky[1])) {
        if (special_index) *special_index = sticky[1] ? (int32_t)sticky[1] - 1 : sidx;
        return fail(B200BPE_ESPECIAL, "text contains a disallowed special token");
    }
    if (rc) return rc;
    if (c.queued > 1) {
        if (run.reruns || (sticky[0] & (ERR_LONGCAP | ERR_MISSCAP | ERR_SLOWCAP)))
            return fail(B200BPE_ECAPACITY, "a work-space had to grow while several device calls were queued: only the last "
                                           "one was re-run, re-issue the others");
        if (sticky[0] & ERR_NOBYTE) return fail(B200BPE_ENOBYTE, "a piece needs a single-byte token that mergeable_ranks does not contain");
        if (sticky[0] & ERR_DOCOFF) return fail(B200BPE_EINVAL, "malformed document offsets in a queued device call");
    }
    if (n_tokens) *n_tokens = S.h_ctr->total_tokens;
    run.lane_per_piece = h->mid_group ? 0 : 1;
    h->publish(run);                      // the last call of a queued series: the counters describe that one
    return B200BPE_OK;
}

extern "C" int b200bpe_device_wait(b200bpe_t *h, uint64_t *n_tokens) { return b200bpe_device_wait_special(h, n_tokens, nullptr); }

extern "C" int b200bpe_encode_device(b200bpe_t *h, const uint8_t *d_text, uint64_t n_bytes, const uint64_t *d_doc_off,
                                     uint64_t n_docs, uint32_t *d_tokens, uint64_t *d_tok_off, uint64_t *n_tokens,
                                     void *stream) {
    int rc = b200bpe_encode_device_async(h, d_text, n_bytes, d_doc_off, n_docs, d_tokens, d_tok_off, nullptr, stream);
    if (rc) return rc;
    return b200bpe_device_wait(h, n_tokens);
}

// A second run of the pipeline over text built on the device (bytes mode, completion search): enqueue, wait, and grow
// and re-run while a work-space was too small.
static int run_again(b200bpe *h, DevCtx *D, Slot &S, const PipeArgs &a, CallStats &run) {
    auto enqueue = [&] { return enqueue_pipeline(h, D, S, a, run); };
    int rc = enqueue();
    return rc ? rc : collect_regrow(S, run, nullptr, nullptr, enqueue);
}

// Bytes mode, a chunk whose run 1 (a1, counters in S.h_ctr and S.h_bytes) found documents that are not well-formed UTF-8: run 2 encodes
// the unstable piece [u_d, end_d) of every such document as one piece, then the splice puts each document's run-1 tokens
// minus the last kdrop[d] in front of its run-2 tokens.  The final tokens and offsets end up in S.w_out / S.w_tokoff and
// *nt is their count.  Run 2 is sized from run 1's counters, which the host already waited for: that is the one extra
// round trip of a damaged chunk.  chunk: run 1's figures, to which the tail runs are added.
static int bytes_tail_runs(b200bpe *h, DevCtx *D, Slot &S, const PipeArgs &a1, uint64_t *nt, CallStats &chunk) {
    const uint64_t n1 = S.h_ctr->total_tokens, drop = S.h_bytes->drop;
    const uint64_t nd = a1.n_docs, tail = S.h_bytes->tail;
    cudaStream_t st = a1.st;
    CUDA_TRY(S.w_b2doc.ensure((size_t)nd + 2)); CUDA_TRY(S.w_b2off.ensure((size_t)nd + 2)); CUDA_TRY(S.w_bbase.ensure((size_t)nd + 2));
    CUDA_TRY(S.w_bpart.ensure((size_t)(nd / SCAN_ITEMS) + 4));
    CUDA_TRY(S.w_btext.ensure((size_t)tail + 64)); CUDA_TRY(S.w_b2out.ensure((size_t)tail + 64));
    if (!S.d_bctr) CUDA_TRY(cudaMalloc((void **)&S.d_bctr, sizeof(Counters)));
    CUDA_TRY(cudaEventRecord(S.ev[14], st));
    CUDA_TRY(enqueue_scan(S.w_btail.p, nd, S.w_bpart.p, S.w_b2doc.p, S.d_bctr, st));
    bytes_gather_kernel<<<(unsigned)((tail + 16 * 256 - 1) / (16 * 256)), 256, 0, st>>>(a1.d_text, nd, S.w_vup.p, S.w_b2doc.p, S.w_btext.p);
    PipeArgs a2;
    a2.d_text = S.w_btext.p; a2.n_bytes = tail; a2.d_doc_off = S.w_b2doc.p; a2.n_docs = nd;
    a2.d_out = S.w_b2out.p; a2.d_tok_off = S.w_b2off.p; a2.st = st; a2.single_piece = true;
    CallStats run2;
    int rc = run_again(h, D, S, a2, run2);
    if (rc) return rc;
    float ms2 = 0; cudaEventElapsedTime(&ms2, S.ev[14], S.ev[4]);
    *nt = n1 - drop + S.h_ctr->total_tokens;
    CUDA_TRY(S.w_bout.ensure((size_t)std::max<uint64_t>(*nt, a1.n_bytes) + 64));
    bytes_count_kernel<<<(unsigned)((nd + 255) / 256), 256, 0, st>>>(S.w_tokoff.p, S.w_b2off.p, S.w_kdrop.p, nd, S.w_btail.p);
    CUDA_TRY(enqueue_scan(S.w_btail.p, nd, S.w_bpart.p, S.w_bbase.p, S.d_bctr, st));
    bytes_splice_kernel<<<(unsigned)std::min<uint64_t>(nd, (uint64_t)D->n_sm * 16), 256, 0, st>>>(
        S.w_out.p, S.w_tokoff.p, S.w_b2out.p, S.w_b2off.p, S.w_kdrop.p, S.w_bbase.p, nd, S.w_bout.p);
    CUDA_TRY(cudaGetLastError());
    std::swap(S.w_out, S.w_bout);
    std::swap(S.w_tokoff, S.w_bbase);
    chunk.ms[4] += ms2;                   // device time of the chunk: run 1, then scan + gather + run 2
    chunk.launches += run2.launches + 9;
    chunk.add_counts(run2);
    return B200BPE_OK;
}

// ---- completion search (b200bpe_encode_with_unstable_batch, kernels_unstable.cuh) ------------------------------------

// byte_pair_encode (src/lib.rs:198-210) of one byte string on the host, through the engine's own pair table: the literal
// loop of _byte_pair_merge (smallest rank, leftmost on ties).  A byte the vocabulary lacks stays a PSEUDO_BASE id.
static void host_byte_pair_encode(const DevTables &T, const std::string &b, std::vector<uint32_t> &ids) {
    const size_t n = b.size();
    ids.resize(n);
    for (size_t j = 0; j < n; j++) ids[j] = T.byte_id[(uint8_t)b[j]];
    std::vector<uint32_t> rk(n);
    auto rank_at = [&](size_t j) { return j + 1 < ids.size() ? pair_lookup(T, ids[j], ids[j + 1]) : RANK_MAX; };
    for (size_t j = 0; j < n; j++) rk[j] = rank_at(j);
    for (;;) {
        uint32_t best = RANK_MAX; size_t bj = 0;
        for (size_t j = 0; j < ids.size(); j++) if (rk[j] < best) { best = rk[j]; bj = j; }
        if (best == RANK_MAX) break;
        ids[bj] = best;                           // the merged token's id is its rank
        ids.erase(ids.begin() + (long)bj + 1); rk.erase(rk.begin() + (long)bj + 1);
        rk[bj] = rank_at(bj);
        if (bj) rk[bj - 1] = rank_at(bj - 1);
    }
}

// The host side of the completion search tables (once per engine, under h->mu).
static void unstable_host_build(b200bpe *h) {
    auto &u = h->uh;
    if (u.built) return;
    const HostTables &H = h->H;
    const DevTables T = H.view();
    u.sorted.clear();
    for (auto &kv : H.decoder) u.sorted.push_back(kv.first);
    std::sort(u.sorted.begin(), u.sorted.end(), [&](uint32_t a, uint32_t b) { return H.decoder.at(a) < H.decoder.at(b); });
    u.lenpre.assign(u.sorted.size() + 1, 0);
    for (size_t i = 0; i < u.sorted.size(); i++) u.lenpre[i + 1] = u.lenpre[i] + H.decoder.at(u.sorted[i]).size();
    u.space.assign((size_t)h->n_ids / 32 + 2, 0);
    u.u8info.assign((size_t)h->n_ids + 1, 0);
    u.ur_idx.assign((size_t)h->n_ids + 1, UR_NONE);
    u.ur_off.assign(1, 0); u.ur_tok.clear();
    u.max_len = 0;
    std::vector<uint32_t> ids, zero;
    for (uint32_t id : u.sorted) {
        const std::string &b = H.decoder.at(id);
        u.max_len = std::max<uint32_t>(u.max_len, (uint32_t)b.size());
        bool all = !b.empty();
        for (char c : b) all &= c == ' ' || c == '\n' || c == '\t';
        if (all) u.space[id >> 5] |= 1u << (id & 31);
        uint32_t c = 0;                           // leading continuation bytes; is the rest well-formed on its own?
        while (c < b.size() && c < 4 && ((uint8_t)b[c] & 0xC0u) == 0x80u) c++;
        bool rest_ok = true;
        if (c < 4) {
            const uint8_t *r = (const uint8_t *)b.data() + c;
            const int64_t rn = (int64_t)b.size() - c;
            zero.assign((size_t)(rn / 32) + 3, 0);
            zero[0] = 1u;                         // one document that starts at byte 0
            for (int64_t w = 0; w * 32 < rn && rest_ok; w++) rest_ok = utf8_bad_word(r, rn, zero.data(), w) == 0;
        }
        u.u8info[id] = (uint8_t)(c | (rest_ok ? 8u : 0u));
        if (b.size() >= 2) {
            host_byte_pair_encode(T, b, ids);
            if (!(ids.size() == 1 && ids[0] == id)) {   // a token its own merges do not reach
                u.ur_idx[id] = (uint32_t)(u.ur_off.size() - 1);
                u.ur_tok.insert(u.ur_tok.end(), ids.begin(), ids.end());
                u.ur_off.push_back((uint32_t)u.ur_tok.size());
            }
        }
    }
    u.built = true;
}

// The device side: one arena per device (under h->mu).
static int unstable_upload(b200bpe *h, DevCtx *D) {
    if (D->d_ut_arena) return B200BPE_OK;
    const auto &u = h->uh;
    struct Part { const void *src; size_t bytes; size_t off; };
    std::vector<uint32_t> one(1, 0);
    Part parts[] = {{u.sorted.data(), u.sorted.size() * 4, 0}, {u.lenpre.data(), u.lenpre.size() * 8, 0},
                    {u.space.data(), u.space.size() * 4, 0}, {u.u8info.data(), u.u8info.size(), 0},
                    {u.ur_idx.data(), u.ur_idx.size() * 4, 0}, {u.ur_off.data(), u.ur_off.size() * 4, 0},
                    {u.ur_tok.empty() ? one.data() : u.ur_tok.data(), std::max<size_t>(u.ur_tok.size(), 1) * 4, 0}};
    size_t total = 0;
    for (auto &p : parts) { p.off = total; total += (p.bytes + 255) & ~(size_t)255; }
    CUDA_TRY(cudaSetDevice(D->device));
    UnstWs &W = D->uw;
    if (!W.d_uc) CUDA_TRY(cudaMalloc((void **)&W.d_uc, sizeof(UnstCounters)));
    if (!W.h_uc) CUDA_TRY(cudaHostAlloc((void **)&W.h_uc, sizeof(UnstCounters), cudaHostAllocPortable));
    if (!W.d_sctr) CUDA_TRY(cudaMalloc((void **)&W.d_sctr, sizeof(Counters)));
    uint8_t *arena = nullptr;
    CUDA_TRY(cudaMalloc((void **)&arena, total));
    for (auto &p : parts)
        if (p.bytes) {
            cudaError_t e = cudaMemcpy(arena + p.off, p.src, p.bytes, cudaMemcpyHostToDevice);
            if (e != cudaSuccess) { cudaFree(arena); return fail(B200BPE_ECUDA, std::string("completion tables: ") + cudaGetErrorString(e)); }
        }
    D->d_ut_arena = arena;
    UnstTables &U = D->ut;
    U.sorted = (const uint32_t *)(arena + parts[0].off); U.n_sorted = (uint32_t)u.sorted.size();
    U.lenpre = (const unsigned long long *)(arena + parts[1].off);
    U.space = (const uint32_t *)(arena + parts[2].off);
    U.u8info = arena + parts[3].off;
    U.ur_idx = (const uint32_t *)(arena + parts[4].off);
    U.ur_off = (const uint32_t *)(arena + parts[5].off);
    U.ur_tok = (const uint32_t *)(arena + parts[6].off);
    U.tok_boff = D->d_tok_boff; U.tok_blob = D->d_tok_blob; U.n_ids = h->n_ids; U.max_len = u.max_len;
    return B200BPE_OK;
}

// grow a buffer that holds `used` elements to at least n, keeping them
template <class Tp>
static cudaError_t grow_keep(DevBuf<Tp> &b, size_t used, size_t n, cudaStream_t st) {
    if (n <= b.cap) return cudaSuccess;
    DevBuf<Tp> nb;
    cudaError_t e = nb.ensure(std::max(n, 2 * b.cap));
    if (e == cudaSuccess && used) e = cudaMemcpyAsync(nb.p, b.p, used * sizeof(Tp), cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { nb.release(); return e; }
    b.release();
    b = nb;
    return cudaSuccess;
}

struct UChunk {                  // one chunk's completions on the host
    std::vector<uint32_t> tok; std::vector<uint64_t> off, grp;   // off: n_comp + 1, grp: n_docs + 1
};

// Completion search of one chunk whose run 1 (a1, with the walk) has been collected: splices the stable tokens (run 1
// minus each document's last L) into S.w_out / S.w_tokoff (*nt = their count), then searches, encodes, truncates and
// deduplicates the candidates in rounds and brings the chunk's completions home.  chunk: run 1's figures; the runs of
// the search add their counts (a deduplication retry counts as a re-run), not their timings or launches.
static int unstable_search(b200bpe *h, DevCtx *D, Slot &S, const PipeArgs &a1, UChunk &out, uint64_t *nt, CallStats &chunk) {
    UnstWs &W = D->uw;
    const UnstTables &U = D->ut;
    const uint64_t nd = a1.n_docs;
    cudaStream_t st = a1.st;
    out.tok.clear(); out.off.assign(1, 0); out.grp.assign((size_t)nd + 1, 0);
    if (nd == 0) return B200BPE_OK;
    const uint64_t n1 = *nt;
    // ---- stable tokens: run 1 minus the last L of every document (the bytes mode's splice with an empty run 2)
    CUDA_TRY(S.w_btail.ensure((size_t)nd + 2)); CUDA_TRY(S.w_bbase.ensure((size_t)nd + 2));
    CUDA_TRY(S.w_bpart.ensure((size_t)(nd / SCAN_ITEMS) + 4));
    CUDA_TRY(S.w_bout.ensure((size_t)std::max<uint64_t>(n1, a1.n_bytes) + 64));
    CUDA_TRY(W.zeros.ensure((size_t)nd + 2));
    if (!S.d_bctr) CUDA_TRY(cudaMalloc((void **)&S.d_bctr, sizeof(Counters)));
    CUDA_TRY(cudaMemsetAsync(W.zeros.p, 0, ((size_t)nd + 2) * 8, st));
    bytes_count_kernel<<<(unsigned)((nd + 255) / 256), 256, 0, st>>>(S.w_tokoff.p, W.zeros.p, S.w_kdrop.p, nd, S.w_btail.p);
    CUDA_TRY(enqueue_scan(S.w_btail.p, nd, S.w_bpart.p, S.w_bbase.p, S.d_bctr, st));
    bytes_splice_kernel<<<(unsigned)std::min<uint64_t>(nd, (uint64_t)D->n_sm * 16), 256, 0, st>>>(
        S.w_out.p, S.w_tokoff.p, S.w_out.p, W.zeros.p, S.w_kdrop.p, S.w_bbase.p, nd, S.w_bout.p);
    std::swap(S.w_out, S.w_bout);
    std::swap(S.w_tokoff, S.w_bbase);
    // ---- search items: (a), the (b) suffixes, (c) per document with unstable bytes
    CUDA_TRY(W.item_base.ensure((size_t)nd + 2));
    CUDA_TRY(W.part.ensure((size_t)(nd / SCAN_ITEMS) + 4));
    CUDA_TRY(cudaMemsetAsync(W.d_uc, 0, sizeof(UnstCounters), st));
    CUDA_TRY(enqueue_scan(S.w_unit.p, nd, W.part.p, W.item_base.p, W.d_sctr, st));
    CUDA_TRY(cudaMemcpyAsync(&W.h_uc->tot[0], W.item_base.p + nd, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&W.h_uc->tot[1], S.w_tokoff.p + nd, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    *nt = W.h_uc->tot[1];
    const uint64_t n_items = W.h_uc->tot[0];
    uint64_t n_cand = 0;
    if (n_items) {
        CUDA_TRY(W.it_lo.ensure((size_t)n_items + 2)); CUDA_TRY(W.it_cnt.ensure((size_t)n_items + 2));
        CUDA_TRY(W.it_bytes.ensure((size_t)n_items + 2)); CUDA_TRY(W.it_doc.ensure((size_t)n_items + 2));
        CUDA_TRY(W.cbase.ensure((size_t)n_items + 2)); CUDA_TRY(W.tbase.ensure((size_t)n_items + 2));
        CUDA_TRY(W.part.ensure((size_t)(n_items / SCAN_ITEMS) + 4));
        unstable_search_kernel<<<(unsigned)((nd * 32 + 255) / 256), 256, 0, st>>>(U, a1.d_text, a1.d_doc_off, nd, S.w_ulen.p,
                                                                                 W.item_base.p, W.it_lo.p, W.it_cnt.p, W.it_bytes.p,
                                                                                 W.it_doc.p, W.d_uc);
        CUDA_TRY(enqueue_scan(W.it_cnt.p, n_items, W.part.p, W.cbase.p, W.d_sctr, st));
        CUDA_TRY(enqueue_scan(W.it_bytes.p, n_items, W.part.p, W.tbase.p, W.d_sctr, st));
        CUDA_TRY(cudaMemcpyAsync(W.h_uc, W.d_uc, sizeof(UnstCounters), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(&W.h_uc->tot[0], W.cbase.p + n_items, 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        if (W.h_uc->err & UERR_BIG) return fail(B200BPE_EINVAL, "the completion candidates of one document need 4 GiB of text or more");
        n_cand = W.h_uc->tot[0];
        chunk.unstable[0] += W.h_uc->n_docs;
    }
    if (n_cand >= 0xFFFFFFF0ull) return fail(B200BPE_EINVAL, "too many completion candidates in one chunk (2^32)");
    UnstItems I;
    I.doc_off = a1.d_doc_off; I.ulen = S.w_ulen.p; I.item_base = W.item_base.p; I.lo = W.it_lo.p; I.cnt = W.it_cnt.p;
    I.doc = W.it_doc.p; I.cbase = W.cbase.p; I.tbase = W.tbase.p; I.n_items = n_items;
    // rounds: at most one chunk of candidate text (B200BPE_CHUNK_MB) and a 32nd of that in candidates
    const uint64_t cap = h->chunk_bytes, max_n = std::max<uint64_t>(cap / 32, 4096);
    CUDA_TRY(W.grp.ensure((size_t)nd + 2)); CUDA_TRY(W.grp_off.ensure((size_t)nd + 2));
    uint64_t n_comp = 0, n_tok = 0, rounds = 0, enc = 0, bpe = 0;
    for (int attempt = 0;; attempt++) {
        uint32_t slots = 4096;
        while (slots < std::min<uint64_t>(2 * n_cand, 1u << 24)) slots <<= 1;
        slots = std::max(slots, W.tslots_min);
        CUDA_TRY(W.tkey.ensure(slots)); CUDA_TRY(W.tidx.ensure(slots)); CUDA_TRY(W.tloc.ensure(slots));
        CUDA_TRY(cudaMemsetAsync(W.tkey.p, 0, (size_t)slots * 8, st));
        CUDA_TRY(cudaMemsetAsync(W.tidx.p, 0xFF, (size_t)slots * 4, st));
        CUDA_TRY(cudaMemsetAsync(W.grp.p, 0, ((size_t)nd + 2) * 4, st));
        UnstTable T{W.tkey.p, W.tidx.p, W.tloc.p, slots - 1};
        const unsigned long long seed = 0x9E3779B97F4A7C15ull * (unsigned long long)(attempt + 1);
        n_comp = n_tok = rounds = enc = bpe = 0;
        uint32_t err = 0;
        for (uint64_t c0 = 0; c0 < n_cand && !err;) {
            CUDA_TRY(cudaMemsetAsync(W.d_uc, 0, sizeof(UnstCounters), st));
            unstable_round_kernel<<<1, 32, 0, st>>>(U, I, n_cand, c0, max_n, cap, W.d_uc);
            CUDA_TRY(cudaMemcpyAsync(&W.h_uc->round, &W.d_uc->round, sizeof(W.h_uc->round), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            const uint64_t c1 = W.h_uc->round[0], nr = c1 - c0;
            CUDA_TRY(W.cinfo.ensure((size_t)nr + 2)); CUDA_TRY(W.o_len.ensure((size_t)nr + 2)); CUDA_TRY(W.s_len.ensure(2 * (size_t)nr + 2));
            CUDA_TRY(W.o_off.ensure((size_t)nr + 2)); CUDA_TRY(W.s_off.ensure(2 * (size_t)nr + 2));
            CUDA_TRY(W.tokoff_o.ensure((size_t)nr + 2)); CUDA_TRY(W.tokoff_s.ensure(2 * (size_t)nr + 2));
            CUDA_TRY(W.nkeep.ensure((size_t)nr + 2)); CUDA_TRY(W.slot.ensure((size_t)nr + 2)); CUDA_TRY(W.keep.ensure((size_t)nr + 2));
            CUDA_TRY(W.kc.ensure((size_t)nr + 2)); CUDA_TRY(W.rcb.ensure((size_t)nr + 2)); CUDA_TRY(W.rtb.ensure((size_t)nr + 2));
            CUDA_TRY(W.part.ensure((size_t)(2 * nr / SCAN_ITEMS) + 4));
            const unsigned grid = (unsigned)((nr + 255) / 256);
            unstable_meta_kernel<<<grid, 256, 0, st>>>(U, I, a1.d_text, c0, nr, W.cinfo.p, W.o_len.p, W.s_len.p, W.d_uc);
            CUDA_TRY(enqueue_scan(W.o_len.p, nr, W.part.p, W.o_off.p, W.d_sctr, st));
            CUDA_TRY(enqueue_scan(W.s_len.p, 2 * nr, W.part.p, W.s_off.p, W.d_sctr, st));
            CUDA_TRY(cudaMemcpyAsync(&W.h_uc->tot[0], W.o_off.p + nr, 8, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaMemcpyAsync(&W.h_uc->tot[1], W.s_off.p + 2 * nr, 8, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            const uint64_t ob = W.h_uc->tot[0], sb = W.h_uc->tot[1];
            // run 2: encode_ordinary of the UTF-8 candidates, single-piece mode for the others and the parts of (c)
            if (ob) {
                CUDA_TRY(W.text_o.ensure((size_t)ob + 64)); CUDA_TRY(W.out_o.ensure((size_t)ob + 64));
                unstable_gather_kernel<<<(unsigned)((ob + 16 * 256 - 1) / (16 * 256)), 256, 0, st>>>(
                    U, a1.d_text, a1.d_doc_off, S.w_ulen.p, W.cinfo.p, nr, 1, W.o_off.p, W.text_o.p);
                PipeArgs a2;
                a2.d_text = W.text_o.p; a2.n_bytes = ob; a2.d_doc_off = W.o_off.p; a2.n_docs = nr;
                a2.d_out = W.out_o.p; a2.d_tok_off = W.tokoff_o.p; a2.st = st;
                CallStats run2;
                int rc = run_again(h, D, S, a2, run2);
                if (rc) return rc;
                chunk.add_counts(run2);
            } else CUDA_TRY(cudaMemsetAsync(W.tokoff_o.p, 0, ((size_t)nr + 1) * 8, st));
            if (sb) {
                CUDA_TRY(W.text_s.ensure((size_t)sb + 64)); CUDA_TRY(W.out_s.ensure((size_t)sb + 64));
                unstable_gather_kernel<<<(unsigned)((sb + 16 * 256 - 1) / (16 * 256)), 256, 0, st>>>(
                    U, a1.d_text, a1.d_doc_off, S.w_ulen.p, W.cinfo.p, nr, 2, W.s_off.p, W.text_s.p);
                PipeArgs a3;
                a3.d_text = W.text_s.p; a3.n_bytes = sb; a3.d_doc_off = W.s_off.p; a3.n_docs = 2 * nr;
                a3.d_out = W.out_s.p; a3.d_tok_off = W.tokoff_s.p; a3.st = st; a3.single_piece = true;
                CallStats run2;
                int rc = run_again(h, D, S, a3, run2);
                if (rc) return rc;
                chunk.add_counts(run2);
            } else CUDA_TRY(cudaMemsetAsync(W.tokoff_s.p, 0, (2 * (size_t)nr + 1) * 8, st));
            // truncate, deduplicate, append
            RunOut R{W.out_o.p, W.tokoff_o.p, W.out_s.p, W.tokoff_s.p};
            UnstResult res{W.res_tok.p, W.res_off.p, W.res_doc.p, W.grp.p};
            CUDA_TRY(cudaMemsetAsync(S.d_bctr, 0, sizeof(Counters), st));
            unstable_insert_kernel<<<grid, 256, 0, st>>>(U, R, W.cinfo.p, S.w_ulen.p, c0, nr, seed, T, W.nkeep.p, W.slot.p, W.d_uc, S.d_bctr);
            unstable_verify_kernel<<<grid, 256, 0, st>>>(U, R, W.cinfo.p, c0, nr, T, res, W.nkeep.p, W.slot.p, W.keep.p, W.kc.p, W.d_uc);
            CUDA_TRY(enqueue_scan(W.keep.p, nr, W.part.p, W.rcb.p, W.d_sctr, st));
            CUDA_TRY(enqueue_scan(W.kc.p, nr, W.part.p, W.rtb.p, W.d_sctr, st));
            CUDA_TRY(cudaMemcpyAsync(W.h_uc, W.d_uc, sizeof(UnstCounters), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaMemcpyAsync(&W.h_uc->tot[0], W.rcb.p + nr, 8, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaMemcpyAsync(&W.h_uc->tot[1], W.rtb.p + nr, 8, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaMemcpyAsync(S.h_ctr, S.d_bctr, sizeof(Counters), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            CUDA_TRY(cudaGetLastError());
            if (S.h_ctr->err & ERR_NOBYTE)
                return fail(B200BPE_ENOBYTE, "a piece needs a single-byte token that mergeable_ranks does not contain");
            err = W.h_uc->err;
            if (err) break;
            enc += W.h_uc->n_encoded; bpe += W.h_uc->n_bpe;
            const uint64_t kept = W.h_uc->tot[0], toks = W.h_uc->tot[1];
            CUDA_TRY(grow_keep(W.res_tok, (size_t)n_tok, (size_t)(n_tok + toks) + 1, st));
            CUDA_TRY(grow_keep(W.res_off, (size_t)(n_comp ? n_comp + 1 : 0), (size_t)(n_comp + kept) + 2, st));
            CUDA_TRY(grow_keep(W.res_doc, (size_t)n_comp, (size_t)(n_comp + kept) + 1, st));
            res = UnstResult{W.res_tok.p, W.res_off.p, W.res_doc.p, W.grp.p};
            unstable_write_kernel<<<grid, 256, 0, st>>>(U, R, W.cinfo.p, nr, T, res, W.keep.p, W.kc.p, W.slot.p, W.rcb.p, W.rtb.p,
                                                        n_comp, n_tok);
            n_comp += kept; n_tok += toks; rounds++;
            c0 = c1;
        }
        if (!err) break;
        if (attempt >= 3) return fail(B200BPE_ECUDA, "completion deduplication did not converge");
        if (err & UERR_TABLE) W.tslots_min = slots * 4;   // else UERR_COLLIDE: the next attempt has another seed
        chunk.reruns++;
    }
    // ---- the chunk's completions: tokens, completion boundaries, per-document ranges
    CUDA_TRY(grow_keep(W.res_off, (size_t)(n_comp ? n_comp + 1 : 0), (size_t)n_comp + 2, st));
    W.h_uc->tot[2] = n_tok;
    CUDA_TRY(cudaMemcpyAsync(W.res_off.p + n_comp, &W.h_uc->tot[2], 8, cudaMemcpyHostToDevice, st));
    CUDA_TRY(enqueue_scan(W.grp.p, nd, W.part.p, W.grp_off.p, W.d_sctr, st));
    out.tok.resize((size_t)n_tok); out.off.resize((size_t)n_comp + 1);
    if (n_tok) CUDA_TRY(cudaMemcpyAsync(out.tok.data(), W.res_tok.p, (size_t)n_tok * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out.off.data(), W.res_off.p, ((size_t)n_comp + 1) * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out.grp.data(), W.grp_off.p, ((size_t)nd + 1) * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    chunk.unstable[1] += enc; chunk.unstable[2] += bpe; chunk.unstable[3] += rounds; chunk.unstable[4] += n_comp;
    return B200BPE_OK;
}

// --------------------------------------------------------------------------------------------
// host path: host buffers in, ONE pinned result out; chunks round-robin over the devices
// --------------------------------------------------------------------------------------------
struct HostJob {
    b200bpe *h = nullptr;
    const uint8_t *text = nullptr; const uint64_t *doc_off = nullptr; uint64_t n_docs = 0;
    bool single_piece = false, pageable = false, bytes = false, unstable = false;
    bool count_only = false;                      // token offsets only: no device token buffer, no token download
    const uint8_t *sp_flags = nullptr;
    const ChunkPlan *plan = nullptr;              // chunk c = parts [cut[c], cut[c+1]) (doc_seams.h)
    const uint64_t *part_off = nullptr;           // the parts' byte offsets: plan->part_off, or doc_off when nothing was cut
    std::vector<std::atomic<long long>> count;    // tokens of chunk c, -1 until its kernels are done
    b200bpe_result *r = nullptr; size_t tok_cap = 0;
    std::atomic<int> error{0}; std::atomic<bool> overflow{false};
    std::string error_msg; std::mutex err_mu;
    int special_idx = -1; uint64_t special_pos = 0;
    CallStats stats; std::mutex stat_mu;          // the workers that finished, merged (under stat_mu)
    std::vector<UChunk> uch;                      // completion search: chunk c's completions

    void set_error(int rc) {
        std::lock_guard<std::mutex> lk(err_mu);
        if (!error.load()) { error_msg = g_last_error; error.store(rc); }
    }
};

// the chunks of one device: c = first, first + step, ...
static void host_worker(HostJob *J, int dev_index, size_t first, size_t step) {
    b200bpe *h = J->h;
    DevCtx *D = h->devs[dev_index];
    const std::vector<uint64_t> &cut = J->plan->cut;
    const size_t n_chunks = cut.size() - 1;
    std::vector<size_t> mine;
    for (size_t c = first; c < n_chunks; c += step) mine.push_back(c);
    auto bail = [&](int rc) {
        if (rc) J->set_error(rc);
        for (size_t k = 0; k < mine.size(); k++) { long long m1 = -1; J->count[mine[k]].compare_exchange_strong(m1, 0); }   // never leave a waiter spinning
        for (int i = 0; i < DevCtx::N_SLOTS; i++) { cudaStreamSynchronize(D->slots[i].up); cudaStreamSynchronize(D->slots[i].stream); }
    };
    if (mine.empty()) return;
    if (cudaSetDevice(D->device) != cudaSuccess) { fail(B200BPE_ECUDA, "cudaSetDevice failed"); return bail(B200BPE_ECUDA); }
    const uint64_t *part_off = J->part_off;
    auto slot_of = [&](size_t k) -> Slot & { return D->slots[k % DevCtx::N_SLOTS]; };

    // Upload of chunk k into its slot.  Pinned caller memory: on the slot's own stream, i.e. behind the download of the
    // slot's previous chunk, so that uploads and downloads do not run free and fight for the link.  Pageable caller
    // memory: helper threads fill a pinned block quarter by quarter and the quarters go up on the slot's UPLOAD stream,
    // which only waits for the kernels (ev[4]) of the slot's previous chunk, so that the host never sits behind a download.
    auto enqueue_h2d = [&](size_t k) -> int {
        Slot &S = slot_of(k);
        const size_t c = mine[k];
        const uint64_t lo = cut[c], hi = cut[c + 1], b0 = part_off[lo], nb = part_off[hi] - b0, nd = hi - lo;
        const bool staged = J->pageable && nb;
        cudaStream_t us = staged ? S.up : S.stream;
        if (!staged || S.w_text.cap < (size_t)nb + 64 || S.w_docoff.cap < (size_t)nd + 2 || S.w_tokoff.cap < (size_t)nd + 2 ||
            (!J->count_only && S.w_out.cap < (size_t)nb + 64))
            CUDA_TRY(cudaStreamSynchronize(S.stream));           // slot free again (or a buffer has to grow: nothing may be in flight)
        else if (k >= (size_t)DevCtx::N_SLOTS) CUDA_TRY(cudaStreamWaitEvent(S.up, S.ev[4], 0));
        CUDA_TRY(S.w_text.ensure((size_t)nb + 64)); CUDA_TRY(S.w_docoff.ensure((size_t)nd + 2));
        CUDA_TRY(S.w_tokoff.ensure((size_t)nd + 2));
        if (!J->count_only) CUDA_TRY(S.w_out.ensure((size_t)nb + 64));
        const uint8_t *src = J->text + b0;
        CUDA_TRY(cudaEventRecord(S.ev[5], us));
        if (staged) {
            CUDA_TRY(cudaStreamSynchronize(S.up));               // the block's previous upload has left it
            if (S.stage.cap < nb) {
                if (S.stage.p) cudaFreeHost(S.stage.p);
                S.stage.p = nullptr; S.stage.cap = 0;
                const size_t want = (size_t)nb + (size_t)(nb / 8) + 4096;
                CUDA_TRY(cudaHostAlloc(&S.stage.p, want, cudaHostAllocPortable));
                S.stage.cap = want;
            }
            uint8_t *stg = (uint8_t *)S.stage.p;
            const size_t group = std::max<size_t>((((size_t)nb / 4) + 4095) & ~(size_t)4095, (size_t)4 << 20);
            for (size_t g0 = 0; g0 < (size_t)nb; g0 += group) {
                const size_t len = std::min(group, (size_t)nb - g0);
                pool_for(h->pool, len, (size_t)1 << 20, [&](size_t lo, size_t hi) { memcpy(stg + g0 + lo, src + g0 + lo, hi - lo); });
                CUDA_TRY(cudaMemcpyAsync(S.w_text.p + g0, stg + g0, len, cudaMemcpyHostToDevice, us));
            }
        } else if (nb) CUDA_TRY(cudaMemcpyAsync(S.w_text.p, src, nb, cudaMemcpyHostToDevice, us));
        CUDA_TRY(cudaMemcpyAsync(S.w_docoff.p, part_off + lo, (nd + 1) * 8, cudaMemcpyHostToDevice, us));
        if (b0) add_offset_kernel<<<(unsigned)((nd + 1 + 255) / 256), 256, 0, us>>>(S.w_docoff.p, nd + 1, -(long long)b0);
        CUDA_TRY(cudaEventRecord(S.ev[6], us));
        if (staged) CUDA_TRY(cudaStreamWaitEvent(S.stream, S.ev[6], 0));     // the slot's pipeline starts when its text has arrived
        return B200BPE_OK;
    };
    auto args_of = [&](size_t k) {
        Slot &S = slot_of(k);
        const size_t c = mine[k];
        const uint64_t lo = cut[c], hi = cut[c + 1];
        PipeArgs a;
        a.d_text = S.w_text.p; a.n_bytes = part_off[hi] - part_off[lo]; a.d_doc_off = S.w_docoff.p; a.n_docs = hi - lo;
        a.d_out = J->count_only ? nullptr : S.w_out.p; a.d_tok_off = S.w_tokoff.p; a.st = S.stream; a.single_piece = J->single_piece; a.sp_flags = J->sp_flags;
        a.bytes = J->bytes; a.unstable = J->unstable;
        return a;
    };
    size_t known = 0; uint64_t known_sum = 0;                    // prefix of the per-chunk token counts seen so far
    std::vector<CallStats> chunk(mine.size());
    CallStats worker;
    // finalise chunk k: wait for its kernels, then send its offsets + tokens home (async) at their final place
    auto drain = [&](size_t k) -> int {
        Slot &S = slot_of(k);
        const size_t c = mine[k];
        const uint64_t lo = cut[c], hi = cut[c + 1], nd = hi - lo;
        CallStats &run = chunk[k];
        int sidx = -1; uint64_t spos = 0;
        int rc = collect_regrow(S, run, &sidx, &spos, [&] { return enqueue_pipeline(h, D, S, args_of(k), run); });
        if (rc == B200BPE_ESPECIAL) {
            std::lock_guard<std::mutex> lk(J->err_mu);
            const uint64_t gpos = spos + part_off[lo];
            if (J->special_idx < 0 || gpos < J->special_pos) { J->special_idx = sidx; J->special_pos = gpos; }
        }
        if (rc) return rc;
        cudaEventElapsedTime(&run.ms[5], S.ev[5], S.ev[6]);
        uint64_t nt = S.h_ctr->total_tokens;
        if (J->bytes && S.h_bytes->n_docs) {                     // documents that are not well-formed UTF-8: run 2 + splice
            run.bytes_repairs += S.h_bytes->n_docs;
            rc = bytes_tail_runs(h, D, S, args_of(k), &nt, run);
            if (rc) return rc;
        }
        if (J->unstable) {                                       // stable tokens + the chunk's completions
            rc = unstable_search(h, D, S, args_of(k), J->uch[c], &nt, run);
            if (rc) return rc;
        }
        const uint8_t head = J->plan->head[c];
        run.seams = head ? 1 : 0; run.docs_cut = head == 2 ? 1 : 0;
        worker.add(run);
        J->count[c].store((long long)nt);
        while (known < c) {                                      // token base = counts of all earlier chunks (other devices)
            long long v = J->count[known].load();
            if (v < 0) {
                if (J->error.load() || J->overflow.load()) return B200BPE_OK;
                std::this_thread::yield();
                continue;
            }
            known_sum += (uint64_t)v; known++;
        }
        const uint64_t token_base = known_sum;
        if (!J->count_only && token_base + nt > J->tok_cap) { J->overflow.store(true); return B200BPE_OK; }
        if (token_base) add_offset_kernel<<<(unsigned)((nd + 1 + 255) / 256), 256, 0, S.stream>>>(S.w_tokoff.p, nd + 1, (long long)token_base);
        CUDA_TRY(cudaEventRecord(S.ev[5], S.stream));
        // the offsets of the documents that start in the chunk (after its first part when that continues a document cut
        // at a seam), and the last chunk's end: every entry of the result is written once, and no seam is
        const uint64_t d0 = J->plan->first_doc[c], d1 = J->plan->first_doc[c + 1] + (c + 1 == n_chunks ? 1 : 0);
        if (d1 > d0)
            CUDA_TRY(cudaMemcpyAsync((uint64_t *)J->r->off.p + d0, S.w_tokoff.p + (head ? 1 : 0), (d1 - d0) * 8,
                                     cudaMemcpyDeviceToHost, S.stream));
        if (nt && !J->count_only)
            CUDA_TRY(cudaMemcpyAsync((uint32_t *)J->r->tok.p + token_base, S.w_out.p, nt * 4, cudaMemcpyDeviceToHost, S.stream));
        CUDA_TRY(cudaEventRecord(S.ev[6], S.stream));
        return B200BPE_OK;
    };
    auto stop = [&]() { return J->error.load() != 0 || J->overflow.load(); };
    // uploads run AHEAD chunks in front of the kernels; the slot of chunk k + AHEAD last served chunk k + AHEAD - N_SLOTS
    // <= k - 2, which was drained (its download issued) in an earlier iteration
    const size_t AHEAD = (size_t)DevCtx::N_SLOTS - 2;
    int rc = B200BPE_OK;
    for (size_t k = 0; k < AHEAD && k < mine.size(); k++) { rc = enqueue_h2d(k); if (rc) return bail(rc); }
    // The completion search of a chunk waits for the device several times per round, so it does not run next to the next
    // chunk's kernels: each chunk is drained before the next one starts (uploads still run ahead).
    const size_t lag = J->unstable ? 0 : 1;
    for (size_t k = 0; k < mine.size() && !stop(); k++) {
        if (k + AHEAD < mine.size()) { rc = enqueue_h2d(k + AHEAD); if (rc) return bail(rc); }
        rc = enqueue_pipeline(h, D, slot_of(k), args_of(k), chunk[k]);
        if (rc) return bail(rc);
        if (k >= lag) { rc = drain(k - lag); if (rc) return bail(rc); }   // overlaps with chunk k's kernels (lag 1)
    }
    if (lag && !stop()) { rc = drain(mine.size() - 1); if (rc) return bail(rc); }
    bail(0);
    if (!stop()) { Slot &S = slot_of(mine.size() - 1); cudaEventElapsedTime(&worker.ms[6], S.ev[5], S.ev[6]); }   // the last D2H
    std::lock_guard<std::mutex> lk(J->stat_mu);
    J->stats.merge(worker);
}

// Chunk plan of the host path (doc_seams.h plan_chunks), with its errors as B200BPE_EINVAL
static int chunk_plan(const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs, size_t chunk, PlanMode mode,
                      const SeamSpecials &sp, ChunkPlan &plan) {
    const int rc = plan_chunks(text, doc_off, n_docs, chunk, mode, sp, plan);
    if (rc == PLAN_UNORDERED) return fail(B200BPE_EINVAL, "document offsets must be non-decreasing");
    if (rc == PLAN_TOO_LARGE)
        return fail(B200BPE_EINVAL, mode == PLAN_SEAMS
                                        ? "a document has a stretch of >= 4 GiB without a seam (a word gap or line start "
                                          "where it may be cut): not supported"
                                        : "a single document of >= 4 GiB is not supported in bytes mode, the completion "
                                          "search, single-piece mode or training");
    return B200BPE_OK;
}

// count_off != NULL: count only, the token offsets go to count_off[0 .. n_docs] and *out is not touched
static int encode_host(b200bpe *h, const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs, bool single_piece,
                       const uint8_t *sp_flags, b200bpe_result **out, int *special_idx, bool bytes = false,
                       b200bpe_result **completions = nullptr, uint64_t *count_off = nullptr) {
    const uint64_t n_bytes = doc_off[n_docs];
    if (doc_off[0] != 0) return fail(B200BPE_EINVAL, "document offsets must start at 0");
    const int n_dev = (int)h->devs.size();
    if (!h->pool) h->pool = new TaskPool();
    h->pool->ensure(h->copy_threads);
    // ---- chunk plan: ranges of parts, i.e. of documents and, for documents larger than a chunk, of their pieces between
    // seams.  Bytes mode and the completion search read each document from its first ill-formed byte or its last piece
    // to its end, so their documents are not cut.
    size_t chunk = h->chunk_bytes;
    if (!h->chunk_forced && n_dev > 1) chunk = std::min<size_t>(64u << 20, std::max<size_t>(8u << 20, (size_t)(n_bytes / (4 * (uint64_t)n_dev))));
    const PlanMode mode = single_piece ? PLAN_WHOLE : (bytes || completions) ? PLAN_DOCS : PLAN_SEAMS;
    SeamSpecials sp;
    sp.str = h->specials.data(); sp.n = h->specials.size(); sp.flags = sp_flags;
    ChunkPlan plan;
    if (int rc = chunk_plan(text, doc_off, n_docs, chunk, mode, sp, plan)) return rc;
    const size_t n_chunks = plan.cut.size() - 1;
    bool pageable = false;
    if (n_bytes) {
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, text) != cudaSuccess) { cudaGetLastError(); pageable = true; }
        else pageable = (at.type == cudaMemoryTypeUnregistered);
    }
    // tokens <= bytes; bytes/2 covers everything but pathological text, which gets a second pass with the worst case
    CallStats redo;                                               // grown, re-runs and token passes of all passes
    for (int pass = 0; pass < 2; pass++) {
        HostJob J;
        J.h = h; J.text = text; J.doc_off = doc_off; J.n_docs = n_docs; J.single_piece = single_piece; J.pageable = pageable;
        J.sp_flags = sp_flags; J.plan = &plan; J.part_off = plan.part_off.empty() ? doc_off : plan.part_off.data(); J.bytes = bytes; J.unstable = completions != nullptr; J.count_only = count_off != nullptr;
        if (J.unstable) J.uch.resize(n_chunks);
        J.count = std::vector<std::atomic<long long>>(n_chunks);
        for (auto &c : J.count) c.store(-1);
        b200bpe_result *r = new b200bpe_result();
        r->owner = h; r->n_docs = n_docs;
        r->off = h->take_pinned((size_t)(n_docs + 1) * 8);
        const size_t want_tok = pass == 0 ? (size_t)(n_bytes / 2) + 4096 : (size_t)n_bytes + 4096;
        if (!J.count_only) r->tok = h->take_pinned(want_tok * 4);
        auto cleanup = [&](int rc) { h->give_pinned(r->tok); h->give_pinned(r->off); delete r; return rc; };
        if (!r->off.p || (!J.count_only && !r->tok.p)) return cleanup(fail(B200BPE_ECUDA, "pinned allocation failed"));
        J.r = r; J.tok_cap = r->tok.cap / 4;
        const int workers = (int)std::min<size_t>((size_t)n_dev, n_chunks);
        if (workers <= 1) host_worker(&J, 0, 0, 1);
        else {
            std::vector<std::thread> th;
            for (int d = 0; d < workers; d++) th.emplace_back(host_worker, &J, d, (size_t)d, (size_t)workers);
            for (auto &t : th) t.join();
        }
        redo.grown |= J.stats.grown; redo.reruns += J.stats.reruns; redo.token_passes = (uint32_t)pass + 1;
        if (J.error.load() || J.overflow.load()) h->publish_redo(redo);
        if (J.error.load()) {
            g_last_error = J.error_msg;
            if (J.error.load() == B200BPE_ESPECIAL && special_idx) *special_idx = J.special_idx;
            return cleanup(J.error.load());
        }
        if (J.overflow.load()) { cleanup(0); continue; }
        uint64_t total = 0;
        for (auto &c : J.count) total += (uint64_t)std::max<long long>(0, c.load());
        r->n_tokens = total;
        J.stats.grown = redo.grown; J.stats.reruns = redo.reruns; J.stats.token_passes = redo.token_passes;
        J.stats.lane_per_piece = h->mid_group ? 0 : 1;
        h->publish(J.stats);
        if (count_off) {
            memcpy(count_off, r->off.p, (size_t)(n_docs + 1) * 8);
            return cleanup(B200BPE_OK);
        }
        if (completions) {                                        // the chunks' completions, back to back
            b200bpe_result *r2 = new b200bpe_result();
            r2->owner = h; r2->on_host_vec = true;
            size_t nt = 0, nc = 0;
            for (auto &u : J.uch) { nt += u.tok.size(); nc += u.off.size() - 1; }
            r2->vtok.reserve(nt); r2->voff.reserve(nc + 1); r2->vgrp.reserve((size_t)n_docs + 1);
            r2->vgrp.push_back(0);
            for (auto &u : J.uch) {
                const uint64_t tb = r2->vtok.size(), cb = r2->voff.size();
                r2->vtok.insert(r2->vtok.end(), u.tok.begin(), u.tok.end());
                for (size_t q = 0; q + 1 < u.off.size(); q++) r2->voff.push_back(tb + u.off[q]);
                for (size_t d = 1; d < u.grp.size(); d++) r2->vgrp.push_back(cb + u.grp[d]);
            }
            r2->voff.push_back(r2->vtok.size());
            r2->n_tokens = r2->vtok.size(); r2->n_docs = r2->voff.size() - 1;
            h->live_results++;
            *completions = r2;
        }
        h->live_results++;                                        // caller holds h->mu
        *out = r;
        return B200BPE_OK;
    }
    return fail(B200BPE_ECUDA, "token buffer sizing did not converge");
}

extern "C" int b200bpe_encode_ordinary_batch(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off,
                                             uint64_t n_docs, b200bpe_result_t **out) {
    if (h) h->reset_stats();
    if (!h || !doc_off || !out) return fail(B200BPE_EINVAL, "null argument");
    if (doc_off[n_docs] && !text) return fail(B200BPE_EINVAL, "null text");
    std::lock_guard<std::mutex> lk(h->mu);
    DeviceGuard guard;
    return encode_host(h, text, doc_off, n_docs, false, nullptr, out, nullptr);
}

// CoreBPE::_encode_bytes (src/py.rs:72-115) for every document of a batch: documents that are well-formed UTF-8 get
// exactly the tokens of b200bpe_encode_ordinary_batch; the others are cut at their first ill-formed byte and repaired on
// the device (kernels_bytes.cuh).
extern "C" int b200bpe_encode_bytes_batch(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs,
                                          b200bpe_result_t **out) {
    if (h) h->reset_stats();
    if (!h || !doc_off || !out) return fail(B200BPE_EINVAL, "null argument");
    if (doc_off[n_docs] && !text) return fail(B200BPE_EINVAL, "null text");
    if (!h->decode_on_device)
        return fail(B200BPE_EINVAL, "bytes mode reads token lengths from the device decode tables: every token id must be < 2^24");
    std::lock_guard<std::mutex> lk(h->mu);
    DeviceGuard guard;
    return encode_host(h, text, doc_off, n_docs, false, nullptr, out, nullptr, true);
}

extern "C" int b200bpe_encode_single_piece(b200bpe_t *h, const uint8_t *piece, uint64_t len, b200bpe_result_t **out) {
    if (h) h->reset_stats();
    if (!h || !out || (len && !piece)) return fail(B200BPE_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(h->mu);
    DeviceGuard guard;
    uint64_t off[2] = {0, len};
    return encode_host(h, piece, off, 1, true, nullptr, out, nullptr);
}

// CoreBPE::encode (src/lib.rs:375-442) + the disallowed-special check of Encoding.encode (tiktoken/core.py:120-124),
// both on the device: one multi-pattern scan finds every occurrence of a special token; a disallowed one is an
// error (the leftmost is reported), allowed ones cut their document into haystacks for the pre-tokeniser and are
// emitted as their own ids.  flags[i]: 1 = allowed, 2 = disallowed, 0 = ordinary text.
extern "C" int b200bpe_encode_batch_special(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs,
                                            const uint8_t *flags, b200bpe_result_t **out, int32_t *special_index) {
    if (h) h->reset_stats();
    if (!h || !doc_off || !out) return fail(B200BPE_EINVAL, "null argument");
    if (doc_off[n_docs] && !text) return fail(B200BPE_EINVAL, "null text");
    std::lock_guard<std::mutex> lk(h->mu);
    DeviceGuard guard;
    int sidx = -1;
    int rc = encode_host(h, text, doc_off, n_docs, false, any_flag(h, flags) ? flags : nullptr, out, &sidx);
    if (rc == B200BPE_ESPECIAL && special_index) *special_index = sidx;
    return rc;
}

// The token offsets of b200bpe_encode_batch_special without the tokens: the pipeline runs up to the count scan, and
// only the sub-tiles that hold a document start are gathered (without token stores); only the offsets come home.
extern "C" int b200bpe_count_batch(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs,
                                   const uint8_t *flags, uint64_t *tok_off, int32_t *special_index) {
    if (h) h->reset_stats();
    if (!h || !doc_off || !tok_off) return fail(B200BPE_EINVAL, "null argument");
    if (doc_off[n_docs] && !text) return fail(B200BPE_EINVAL, "null text");
    std::lock_guard<std::mutex> lk(h->mu);
    DeviceGuard guard;
    int sidx = -1;
    int rc = encode_host(h, text, doc_off, n_docs, false, any_flag(h, flags) ? flags : nullptr, nullptr, &sidx, false, nullptr, tok_off);
    if (rc == B200BPE_ESPECIAL && special_index) *special_index = sidx;
    return rc;
}

extern "C" int b200bpe_encode_batch(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs,
                                    const uint8_t *allowed, b200bpe_result_t **out) {
    if (!h) return fail(B200BPE_EINVAL, "null argument");
    h->reset_stats();
    std::vector<uint8_t> flags(h->specials.size() + 1, 0);
    if (allowed) for (size_t i = 0; i < h->specials.size(); i++) flags[i] = allowed[i] ? 1 : 0;
    return b200bpe_encode_batch_special(h, text, doc_off, n_docs, allowed ? flags.data() : nullptr, out, nullptr);
}

// Encoding.encode_with_unstable (tiktoken/core.py:208-243 -> src/py.rs:117-131 -> CoreBPE::_encode_unstable_native,
// src/lib.rs:483-599) for every document of a batch, the disallowed check included; kernels_unstable.cuh.
extern "C" int b200bpe_encode_with_unstable_batch(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs,
                                                  const uint8_t *flags, b200bpe_result_t **stable,
                                                  b200bpe_result_t **completions, int32_t *special_index) {
    if (h) h->reset_stats();
    if (!h || !doc_off || !stable || !completions) return fail(B200BPE_EINVAL, "null argument");
    if (doc_off[n_docs] && !text) return fail(B200BPE_EINVAL, "null text");
    if (!h->decode_on_device)
        return fail(B200BPE_EINVAL, "the completion search reads token bytes from the device decode tables: every token id must be < 2^24");
    std::lock_guard<std::mutex> lk(h->mu);
    DeviceGuard guard;
    unstable_host_build(h);
    for (auto *D : h->devs) { int rc = unstable_upload(h, D); if (rc) return rc; }
    int sidx = -1;
    b200bpe_result *comp = nullptr;
    int rc = encode_host(h, text, doc_off, n_docs, false, any_flag(h, flags) ? flags : nullptr, stable, &sidx, false, &comp);
    if (rc == B200BPE_ESPECIAL && special_index) *special_index = sidx;
    if (!rc) *completions = comp;
    return rc;
}

extern "C" const char *b200bpe_special_name(b200bpe_t *h, int32_t index) {
    if (!h || index < 0 || (size_t)index >= h->specials.size()) return nullptr;
    return h->specials[(size_t)index].c_str();
}

extern "C" const uint32_t *b200bpe_result_tokens(const b200bpe_result_t *r) {
    return r->on_host_vec ? r->vtok.data() : (const uint32_t *)r->tok.p;
}
extern "C" const uint64_t *b200bpe_result_offsets(const b200bpe_result_t *r) {
    return r->on_host_vec ? r->voff.data() : (const uint64_t *)r->off.p;
}
extern "C" const uint64_t *b200bpe_result_groups(const b200bpe_result_t *r, uint64_t *n_groups) {
    if (n_groups) *n_groups = r->vgrp.empty() ? 0 : r->vgrp.size() - 1;
    return r->vgrp.empty() ? nullptr : r->vgrp.data();
}
extern "C" uint64_t b200bpe_result_n_tokens(const b200bpe_result_t *r) { return r->n_tokens; }
extern "C" uint64_t b200bpe_result_n_docs(const b200bpe_result_t *r) { return r->n_docs; }
extern "C" void b200bpe_result_free(b200bpe_result_t *r) {
    if (!r) return;
    b200bpe *h = r->owner;
    bool last = false;
    if (h) {
        std::lock_guard<std::mutex> lk(h->mu);
        if (!r->on_host_vec) { h->give_pinned(r->tok); h->give_pinned(r->off); }
        h->live_results--;
        last = h->dead && h->live_results == 0;
    }
    delete r;
    if (last) engine_teardown(h);
}

// --------------------------------------------------------------------------------------------
// decode
// --------------------------------------------------------------------------------------------
static const std::string *decode_one(b200bpe *h, uint32_t t) {
    auto it = h->H.decoder.find(t);
    if (it != h->H.decoder.end()) return &it->second;
    auto it2 = h->special_decoder.find(t);
    if (it2 != h->special_decoder.end()) return &it2->second;
    return nullptr;
}

extern "C" int b200bpe_decode_bytes(b200bpe_t *h, const uint32_t *tokens, uint64_t n_tokens, uint8_t *out,
                                    uint64_t out_cap, uint64_t *out_len, uint32_t *bad_token) {
    if (!h || (n_tokens && !tokens) || !out_len) return fail(B200BPE_EINVAL, "null argument");
    uint64_t k = 0;
    for (uint64_t i = 0; i < n_tokens; i++) {
        const std::string *s = decode_one(h, tokens[i]);
        if (!s) {
            if (bad_token) *bad_token = tokens[i];
            return fail(B200BPE_EKEY, "Invalid token for decoding: " + std::to_string(tokens[i]));
        }
        if (out && k + s->size() <= out_cap) memcpy(out + k, s->data(), s->size());
        k += s->size();
    }
    *out_len = k;
    return B200BPE_OK;
}

// Batched CoreBPE::decode_bytes (src/lib.rs:345-358) on the device: tokens of all documents
// concatenated + per-document token offsets (HOST buffers) -> bytes of all documents concatenated
// + per-document byte offsets.  The result object reuses b200bpe_result: "tokens" holds the bytes
// (n_tokens = byte count), "offsets" the byte offsets.
extern "C" int b200bpe_decode_batch(b200bpe_t *h, const uint32_t *tokens, const uint64_t *tok_off, uint64_t n_docs,
                                    b200bpe_result_t **out, uint32_t *bad_token) {
    if (!h || !tok_off || !out) return fail(B200BPE_EINVAL, "null argument");
    const uint64_t n = tok_off[n_docs];
    if (n && !tokens) return fail(B200BPE_EINVAL, "null tokens");
    if (tok_off[0] != 0) return fail(B200BPE_EINVAL, "token offsets must start at 0");
    for (uint64_t d = 0; d < n_docs; d++)
        if (tok_off[d + 1] < tok_off[d]) return fail(B200BPE_EINVAL, "token offsets must be non-decreasing");
    std::lock_guard<std::mutex> lk(h->mu);
    DeviceGuard guard;
    struct ResultGuard {               // no leak on the error paths below
        b200bpe *h; b200bpe_result *r = nullptr; bool keep = false;
        ~ResultGuard() { if (r && !keep) { h->give_pinned(r->tok); h->give_pinned(r->off); delete r; } }
    } rg{h};
    if (!h->decode_on_device) {        // ids of 2^24 and above exist: host maps (same results)
        b200bpe_result *r = new b200bpe_result();
        rg.r = r;
        r->owner = h; r->n_docs = n_docs;
        uint64_t total = 0;
        for (uint64_t i = 0; i < n; i++) {
            const std::string *s = decode_one(h, tokens[i]);
            if (!s) { if (bad_token) *bad_token = tokens[i]; return fail(B200BPE_EKEY, "Invalid token for decoding: " + std::to_string(tokens[i])); }
            total += s->size();
        }
        r->off = h->take_pinned((size_t)(n_docs + 1) * 8);
        r->tok = h->take_pinned((size_t)total + 16);
        if (!r->off.p || !r->tok.p) return fail(B200BPE_ECUDA, "pinned allocation failed");
        uint8_t *dst = (uint8_t *)r->tok.p; uint64_t k = 0;
        for (uint64_t d = 0; d < n_docs; d++) {
            ((uint64_t *)r->off.p)[d] = k;
            for (uint64_t i = tok_off[d]; i < tok_off[d + 1]; i++) { const std::string *s = decode_one(h, tokens[i]); memcpy(dst + k, s->data(), s->size()); k += s->size(); }
        }
        ((uint64_t *)r->off.p)[n_docs] = k;
        r->n_tokens = k; rg.keep = true; h->live_results++;
        h->publish_timings(CallStats());
        *out = r;
        return B200BPE_OK;
    }
    DevCtx *D = h->devs[0];
    CUDA_TRY(cudaSetDevice(D->device));
    Slot &S = D->slots[0];
    cudaStream_t st = S.stream;
    // reuse slot-0 workspace: w_out = tokens, w_sub_count = lengths, w_sub_base = byte base, w_text = bytes out
    CUDA_TRY(S.w_out.ensure((size_t)n + 4)); CUDA_TRY(S.w_sub_count.ensure((size_t)n + 4));
    CUDA_TRY(S.w_sub_base.ensure((size_t)n + 4)); CUDA_TRY(S.w_scan_part.ensure((size_t)(n / SCAN_ITEMS) + 4));
    CUDA_TRY(S.w_docoff.ensure((size_t)n_docs + 2)); CUDA_TRY(S.w_tokoff.ensure((size_t)n_docs + 2));
    CUDA_TRY(cudaMemsetAsync(S.d_ctr, 0, sizeof(Counters), st));
    CUDA_TRY(cudaMemsetAsync(&S.d_ctr->ticket, 0xFF, sizeof(unsigned int), st));
    CUDA_TRY(cudaEventRecord(S.ev[0], st));
    if (n) CUDA_TRY(cudaMemcpyAsync(S.w_out.p, tokens, n * 4, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(S.w_docoff.p, tok_off, (n_docs + 1) * 8, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaEventRecord(S.ev[1], st));
    if (n) decode_len_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(S.w_out.p, n, D->d_tok_boff, h->n_ids, S.w_sub_count.p, S.d_ctr);
    CUDA_TRY(enqueue_scan(S.w_sub_count.p, n, S.w_scan_part.p, S.w_sub_base.p, S.d_ctr, st));
    CUDA_TRY(cudaMemcpyAsync(S.h_ctr, S.d_ctr, sizeof(Counters), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (S.h_ctr->err & ERR_BADTOKEN) {
        const uint32_t t = tokens[S.h_ctr->ticket];
        if (bad_token) *bad_token = t;
        return fail(B200BPE_EKEY, "Invalid token for decoding: " + std::to_string(t));
    }
    const uint64_t n_out = S.h_ctr->total_tokens;
    CUDA_TRY(S.w_text.ensure((size_t)n_out + 64));
    if (n) decode_copy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(S.w_out.p, n, D->d_tok_boff, h->n_ids, D->d_tok_blob,
                                                                        S.w_sub_base.p, S.w_text.p);
    decode_doc_off_kernel<<<(unsigned)((n_docs + 1 + 255) / 256), 256, 0, st>>>(S.w_docoff.p, n_docs, S.w_sub_base.p, S.w_tokoff.p);
    CUDA_TRY(cudaEventRecord(S.ev[2], st));
    b200bpe_result *r = new b200bpe_result();
    rg.r = r;
    r->owner = h; r->n_docs = n_docs; r->n_tokens = n_out;
    r->off = h->take_pinned((size_t)(n_docs + 1) * 8);
    r->tok = h->take_pinned((size_t)n_out + 16);
    if (!r->off.p || !r->tok.p) return fail(B200BPE_ECUDA, "pinned allocation failed");
    CUDA_TRY(cudaMemcpyAsync(r->off.p, S.w_tokoff.p, (n_docs + 1) * 8, cudaMemcpyDeviceToHost, st));
    if (n_out) CUDA_TRY(cudaMemcpyAsync(r->tok.p, S.w_text.p, n_out, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaEventRecord(S.ev[3], st));
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    CallStats run;
    cudaEventElapsedTime(&run.ms[5], S.ev[0], S.ev[1]);
    cudaEventElapsedTime(&run.ms[4], S.ev[1], S.ev[2]);
    cudaEventElapsedTime(&run.ms[6], S.ev[2], S.ev[3]);
    run.launches = 6;
    h->publish_timings(run);
    rg.keep = true;
    h->live_results++;
    *out = r;
    return B200BPE_OK;
}

extern "C" int b200bpe_last_timings(b200bpe_t *h, float *ms9, uint32_t *n_launches) {
    if (!h) return fail(B200BPE_EINVAL, "null handle");
    const CallStats s = h->stats();
    if (ms9) memcpy(ms9, s.ms, sizeof(s.ms));
    if (n_launches) *n_launches = s.launches;
    return B200BPE_OK;
}

extern "C" int b200bpe_last_reruns(b200bpe_t *h, uint32_t *grown, uint32_t *reruns, uint32_t *token_passes) {
    if (!h) return fail(B200BPE_EINVAL, "null handle");
    const CallStats s = h->stats();
    if (grown) *grown = s.grown;
    if (reruns) *reruns = s.reruns;
    if (token_passes) *token_passes = s.token_passes;
    return B200BPE_OK;
}

extern "C" int b200bpe_last_piece_classes(b200bpe_t *h, uint64_t *counts8, int *lane_per_piece) {
    if (!h) return fail(B200BPE_EINVAL, "null handle");
    const CallStats s = h->stats();
    if (counts8) for (int c = 0; c < N_CLS; c++) counts8[c] = s.cls[c];
    if (lane_per_piece) *lane_per_piece = s.lane_per_piece;
    return B200BPE_OK;
}

extern "C" int b200bpe_last_miss_memo(b200bpe_t *h, uint64_t *misses, uint64_t *merged, uint64_t *unplaced) {
    if (!h) return fail(B200BPE_EINVAL, "null handle");
    const CallStats s = h->stats();
    if (misses) *misses = s.memo[0];
    if (merged) *merged = s.memo[1];
    if (unplaced) *unplaced = s.memo[2];
    return B200BPE_OK;
}

extern "C" int b200bpe_last_bytes_repairs(b200bpe_t *h, uint64_t *n_docs_repaired) {
    if (!h) return fail(B200BPE_EINVAL, "null handle");
    if (n_docs_repaired) *n_docs_repaired = h->stats().bytes_repairs;
    return B200BPE_OK;
}

extern "C" int b200bpe_last_unstable(b200bpe_t *h, uint64_t *stats5) {
    if (!h || !stats5) return fail(B200BPE_EINVAL, "null argument");
    const CallStats s = h->stats();
    for (int i = 0; i < 5; i++) stats5[i] = s.unstable[i];
    return B200BPE_OK;
}

extern "C" int b200bpe_last_doc_seams(b200bpe_t *h, uint64_t *seams, uint64_t *docs_cut) {
    if (!h) return fail(B200BPE_EINVAL, "null handle");
    const CallStats s = h->stats();
    if (seams) *seams = s.seams;
    if (docs_cut) *docs_cut = s.docs_cut;
    return B200BPE_OK;
}

extern "C" int b200bpe_table_bytes(b200bpe_t *h, uint64_t *bytes4) {
    if (!h || !bytes4) return fail(B200BPE_EINVAL, "null argument");
    memcpy(bytes4, h->table_bytes, sizeof(h->table_bytes));
    return B200BPE_OK;
}

// --------------------------------------------------------------------------------------------
// BPE training (tiktoken/_educational.py:119-185 `bpe_train`), kernels_train.cuh
// --------------------------------------------------------------------------------------------
namespace {

struct TrainRun {                              // everything one b200bpe_bpe_train call allocates on its device
    DevBuf<uint8_t> all, ct, uc;
    DevBuf<unsigned long long> doff, npieces, wkey, wcnt, wfirst, wused, part, tbase, dfirst, dcnt, woff;
    DevBuf<unsigned long long> pkey, pcnt, th, tpw, tlen;
    DevBuf<uint32_t> dbits, sfd, pbits, psum, slow, wlen, fbits, tcnt, dlen, wl1, sym, pocc, tslot, stamp, aff, merges;
    Counters *ctr = nullptr, *h_ctr = nullptr; TrainState *st = nullptr, *h_st = nullptr;
    unsigned long long *h_u64 = nullptr;
    cudaStream_t s = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaGraphExec_t exec = nullptr; cudaGraph_t graph = nullptr;
    ~TrainRun() {
        DevBuf<uint8_t> *b8[] = {&all, &ct, &uc};
        for (auto *b : b8) b->release();
        DevBuf<unsigned long long> *b64[] = {&doff, &npieces, &wkey, &wcnt, &wfirst, &wused, &part, &tbase, &dfirst, &dcnt, &woff,
                                             &pkey, &pcnt, &th, &tpw, &tlen};
        for (auto *b : b64) b->release();
        DevBuf<uint32_t> *b32[] = {&dbits, &sfd, &pbits, &psum, &slow, &wlen, &fbits, &tcnt, &dlen, &wl1, &sym, &pocc, &tslot,
                                   &stamp, &aff, &merges};
        for (auto *b : b32) b->release();
        if (ctr) cudaFree(ctr);
        if (st) cudaFree(st);
        if (h_ctr) cudaFreeHost(h_ctr);
        if (h_st) cudaFreeHost(h_st);
        if (h_u64) cudaFreeHost(h_u64);
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
        for (auto &e : ev) if (e) cudaEventDestroy(e);
        if (s) cudaStreamDestroy(s);
    }
};

uint64_t train_pow2(uint64_t x) { uint64_t p = 1; while (p < x) p <<= 1; return p; }

float event_ms(cudaEvent_t a, cudaEvent_t b) { float ms = 0.f; if (cudaEventElapsedTime(&ms, a, b) != cudaSuccess) { cudaGetLastError(); ms = 0.f; } return ms; }

}  // namespace

// make the piece table hold `need` slots at half load, keeping what it holds
static int train_words_reserve(TrainRun &T, TrainWords &W, uint64_t need) {
    const uint64_t want = train_pow2(std::max<uint64_t>(2 * need, 1u << 16));
    if (W.key && W.mask + 1 >= want) return B200BPE_OK;
    TrainRun O;                                           // the old table moves here and is freed on return
    std::swap(O.wkey, T.wkey); std::swap(O.wcnt, T.wcnt); std::swap(O.wfirst, T.wfirst); std::swap(O.wlen, T.wlen);
    const uint64_t n_old = W.key ? W.mask + 1 : 0;
    CUDA_TRY(T.wkey.ensure(want)); CUDA_TRY(T.wcnt.ensure(want)); CUDA_TRY(T.wfirst.ensure(want)); CUDA_TRY(T.wlen.ensure(want));
    CUDA_TRY(cudaMemsetAsync(T.wkey.p, 0, want * 8, T.s)); CUDA_TRY(cudaMemsetAsync(T.wcnt.p, 0, want * 8, T.s));
    CUDA_TRY(cudaMemsetAsync(T.wfirst.p, 0xFF, want * 8, T.s));
    TrainWords N{T.wkey.p, T.wcnt.p, T.wfirst.p, T.wlen.p, want - 1, T.wused.p};
    if (n_old) {
        CUDA_TRY(cudaMemsetAsync(T.wused.p, 0, 8, T.s));
        TrainWords Wo{O.wkey.p, O.wcnt.p, O.wfirst.p, O.wlen.p, W.mask, W.n_used};
        train_rehash_kernel<<<1024, 256, 0, T.s>>>(Wo, n_old, N);
        CUDA_TRY(cudaStreamSynchronize(T.s));
    }
    W = N;
    return B200BPE_OK;
}

extern "C" int b200bpe_bpe_train(const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs, const char *pat_str,
                                 uint32_t vocab_size, int device, uint32_t *merges_out, uint64_t merges_cap,
                                 uint64_t *n_merges_out, double *stats8) {
    if (stats8) for (int i = 0; i < 8; i++) stats8[i] = 0.0;
    if (n_merges_out) *n_merges_out = 0;
    if (!doc_off || !pat_str || !n_merges_out || (merges_cap && !merges_out)) return fail(B200BPE_EINVAL, "null argument");
    const int pattern = pattern_of(pat_str);
    if (pattern < 0) return B200BPE_EPATTERN;
    if (vocab_size < 256) return fail(B200BPE_EINVAL, "vocab_size must be at least 256, so we can encode all bytes");
    if (doc_off[0] != 0) return fail(B200BPE_EINVAL, "document offsets must start at 0");
    const uint64_t N = doc_off[n_docs];
    if (N && !text) return fail(B200BPE_EINVAL, "null text");
    size_t chunk = env_chunk_bytes();
    if (!chunk) chunk = 64u << 20;
    ChunkPlan plan;                                         // the words of a document are counted whole: no seams
    if (int rc = chunk_plan(text, doc_off, n_docs, chunk, PLAN_DOCS, SeamSpecials(), plan)) return rc;
    const std::vector<uint64_t> &cut = plan.cut;
    const uint32_t target = vocab_size;
    if (target == 256) return B200BPE_OK;                  // the 256 single bytes, no merge
    if (merges_cap > 0xFFFFFFF0ull) merges_cap = 0xFFFFFFF0ull;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(B200BPE_ECUDA, "no CUDA device: libb200bpe has no CPU fallback"); }
    if (device < 0 || device >= ndev) return fail(B200BPE_EINVAL, "bad device index");
    DeviceGuard guard;
    CUDA_TRY(cudaSetDevice(device));
    int n_sm = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, device));
    TrainRun T;
    CUDA_TRY(cudaStreamCreateWithFlags(&T.s, cudaStreamNonBlocking));
    for (auto &e : T.ev) CUDA_TRY(cudaEventCreate(&e));
    CUDA_TRY(cudaMalloc((void **)&T.ctr, sizeof(Counters))); CUDA_TRY(cudaMalloc((void **)&T.st, sizeof(TrainState)));
    CUDA_TRY(cudaHostAlloc((void **)&T.h_ctr, sizeof(Counters), cudaHostAllocPortable));
    CUDA_TRY(cudaHostAlloc((void **)&T.h_st, sizeof(TrainState), cudaHostAllocPortable));
    CUDA_TRY(cudaHostAlloc((void **)&T.h_u64, 4 * 8, cudaHostAllocPortable));
    cudaStream_t s = T.s;
    // Unicode class tables of the pre-tokeniser (the engine keeps them in its table arena)
    UcTables uc;
    {
        uint8_t ascii[128];
        uc_ascii_table(ascii);
        const size_t o2 = (sizeof(UC_STAGE1) + 255) & ~(size_t)255, o3 = o2 + ((sizeof(UC_STAGE2) + 255) & ~(size_t)255);
        CUDA_TRY(T.uc.ensure(o3 + 128));
        CUDA_TRY(cudaMemcpy(T.uc.p, UC_STAGE1, sizeof(UC_STAGE1), cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(T.uc.p + o2, UC_STAGE2, sizeof(UC_STAGE2), cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(T.uc.p + o3, ascii, 128, cudaMemcpyHostToDevice));
        uc.stage1 = (const uint16_t *)T.uc.p; uc.stage2 = T.uc.p + o2; uc.ascii = T.uc.p + o3; uc.one = 1u;
    }
    // the corpus stays on the device: each piece is compared with the first occurrence of its word
    CUDA_TRY(T.all.ensure(N + 64));
    if (N) CUDA_TRY(cudaMemcpy(T.all.p, text, N, cudaMemcpyHostToDevice));
    CUDA_TRY(T.fbits.ensure((N + 1 + 1023) / 1024 * 32 + 64));
    CUDA_TRY(cudaMemsetAsync(T.fbits.p, 0, T.fbits.cap * 4, s));
    CUDA_TRY(cudaMemsetAsync(T.st, 0, sizeof(TrainState), s));
    CUDA_TRY(T.npieces.ensure(1)); CUDA_TRY(T.wused.ensure(1));
    CUDA_TRY(cudaMemsetAsync(T.wused.p, 0, 8, s));
    TrainWords W{}; W.n_used = T.wused.p;
    if (int rc = train_words_reserve(T, W, 1u << 15)) return rc;
    double ms_split = 0, ms_words = 0, ms_loop = 0;
    uint64_t n_pieces = 0;
    // ---- split + distinct words, chunk by chunk --------------------------------------------------------------------
    for (size_t c = 0; c + 1 < cut.size(); c++) {
        const uint64_t lo = cut[c], hi = cut[c + 1], base = doc_off[lo], n = doc_off[hi] - base, nd = hi - lo;
        if (n == 0) continue;
        const long long n_words = (long long)((n + 1 + 31) / 32);
        std::vector<unsigned long long> rel(nd + 1);
        for (uint64_t d = 0; d <= nd; d++) rel[d] = doc_off[lo + d] - base;
        CUDA_TRY(T.doff.ensure(nd + 1)); CUDA_TRY(T.ct.ensure(n + 64));
        CUDA_TRY(T.dbits.ensure((size_t)n_words + 8)); CUDA_TRY(T.sfd.ensure((size_t)n_words + 4));
        CUDA_TRY(T.pbits.ensure((size_t)n_words + 8)); CUDA_TRY(T.psum.ensure((size_t)(n_words >> 5) + 4));
        CUDA_TRY(T.slow.ensure(n + 64));                   // every position: the slow list cannot overflow
        CUDA_TRY(cudaMemcpyAsync(T.doff.p, rel.data(), (nd + 1) * 8, cudaMemcpyHostToDevice, s));
        CUDA_TRY(cudaMemcpyAsync(T.ct.p, T.all.p + base, n, cudaMemcpyDeviceToDevice, s));   // 16-byte aligned chunk text
        CUDA_TRY(cudaMemsetAsync(T.ct.p + n, 0, 64, s));
        CUDA_TRY(cudaMemsetAsync(T.ctr, 0, sizeof(Counters), s));
        CUDA_TRY(cudaMemsetAsync(T.dbits.p, 0, ((size_t)n_words + 8) * 4, s));
        CUDA_TRY(cudaMemsetAsync(T.sfd.p, 0xFF, ((size_t)n_words + 4) * 4, s));
        CUDA_TRY(cudaMemsetAsync(T.pbits.p + n_words, 0, 8 * 4, s));
        CUDA_TRY(cudaMemsetAsync(T.npieces.p, 0, 8, s));
        CUDA_TRY(cudaEventRecord(T.ev[0], s));
        mark_docs_kernel<<<(unsigned)((nd + 1 + 255) / 256), 256, 0, s>>>(T.doff.p, nd, n, T.dbits.p, T.sfd.p, nullptr, T.ctr);
        const unsigned grid = (unsigned)((n_words + 255) / 256);
        enqueue_pretok(pattern, false, n_sm, s, T.ct.p, (long long)n, T.dbits.p, uc, T.pbits.p, T.psum.p, n_words, nullptr,
                       T.slow.p, (uint32_t)std::min<uint64_t>(n + 64, 0xFFFFFFF0u), T.ctr);
        CUDA_TRY(cudaEventRecord(T.ev[1], s));
        train_count_kernel<<<grid, 256, 0, s>>>(T.pbits.p, (long long)n, n_words, T.npieces.p);
        CUDA_TRY(cudaMemcpyAsync(T.h_ctr, T.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaMemcpyAsync(T.h_u64, T.npieces.p, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaMemcpyAsync(T.h_u64 + 1, T.wused.p, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        if (T.h_ctr->err & ERR_DOCOFF) return fail(B200BPE_EINVAL, "malformed document offsets");
        if (T.h_ctr->err) return fail(B200BPE_ECUDA, "pre-tokeniser error flags " + std::to_string(T.h_ctr->err));
        n_pieces += T.h_u64[0];
        ms_split += event_ms(T.ev[0], T.ev[1]);
        if (int rc = train_words_reserve(T, W, T.h_u64[0] + T.h_u64[1])) return rc;
        CUDA_TRY(cudaEventRecord(T.ev[2], s));
        train_insert_kernel<<<grid, 256, 0, s>>>(T.ct.p, (long long)n, T.pbits.p, n_words, base, W);
        train_verify_kernel<<<grid, 256, 0, s>>>(T.ct.p, (long long)n, T.pbits.p, n_words, base, W, T.all.p, T.fbits.p, T.st);
        CUDA_TRY(cudaEventRecord(T.ev[3], s));
        CUDA_TRY(cudaStreamSynchronize(s));
        ms_words += event_ms(T.ev[2], T.ev[3]);
    }
    CUDA_TRY(cudaGetLastError());
    // ---- words in order of first occurrence: CSR of symbol ids ----------------------------------------------------
    CUDA_TRY(cudaEventRecord(T.ev[2], s));
    const long long n_tiles = (long long)((N + 1 + 1023) / 1024);
    CUDA_TRY(T.tcnt.ensure((size_t)n_tiles + 4)); CUDA_TRY(T.tbase.ensure((size_t)n_tiles + 4));
    CUDA_TRY(T.part.ensure((size_t)(n_tiles / SCAN_ITEMS) + 4));
    CUDA_TRY(cudaMemsetAsync(T.ctr, 0, sizeof(Counters), s));
    train_tile_count_kernel<<<(unsigned)((n_tiles + 255) / 256), 256, 0, s>>>(T.fbits.p, n_tiles, T.tcnt.p);
    CUDA_TRY(enqueue_scan(T.tcnt.p, (uint64_t)n_tiles, T.part.p, T.tbase.p, T.ctr, s));
    CUDA_TRY(cudaMemcpyAsync(T.h_ctr, T.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(T.h_u64 + 1, T.wused.p, 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    const uint64_t D = T.h_ctr->total_tokens;
    if (D != T.h_u64[1]) return fail(B200BPE_ECUDA, "internal: distinct words and first occurrences disagree");
    if (D >= 0xFFFFFFF0ull) return fail(B200BPE_EINVAL, "too many distinct words (>= 2^32)");
    CUDA_TRY(T.dfirst.ensure(D + 2)); CUDA_TRY(T.dlen.ensure(D + 2)); CUDA_TRY(T.dcnt.ensure(D + 2)); CUDA_TRY(T.wl1.ensure(D + 2));
    CUDA_TRY(T.woff.ensure(D + 2));
    train_compact_kernel<<<n_sm * 8, 256, 0, s>>>(W, T.fbits.p, T.tbase.p, T.dfirst.p, T.dlen.p, T.dcnt.p, T.wl1.p, D, T.st);
    CUDA_TRY(T.part.ensure((size_t)((D + SCAN_ITEMS - 1) / SCAN_ITEMS) + 4));
    CUDA_TRY(cudaMemsetAsync(T.ctr, 0, sizeof(Counters), s));
    CUDA_TRY(enqueue_scan(T.wl1.p, D, T.part.p, T.woff.p, T.ctr, s));
    CUDA_TRY(cudaMemcpyAsync(T.h_ctr, T.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(T.h_st, T.st, sizeof(TrainState), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    if (T.h_st->err) return fail(B200BPE_ECUDA, T.h_st->err & 1u ? "internal: two different pieces share a 64-bit hash"
                                                                 : "internal: word index out of range");
    const uint64_t S = T.h_ctr->total_tokens;               // symbol slots: every word plus its separator
    CUDA_TRY(T.sym.ensure(S + 4));
    if (D) train_fill_kernel<<<n_sm * 8, 256, 0, s>>>(T.all.p, T.dfirst.p, T.dlen.p, T.woff.p, D, T.sym.p);
    CUDA_TRY(cudaStreamSynchronize(s));
    T.all.release(); T.ct.release(); T.slow.release(); T.pbits.release(); T.dbits.release(); T.sfd.release();
    T.wkey.release(); T.wcnt.release(); T.wfirst.release(); T.wlen.release();
    // pair table: distinct keys <= P0 initial pairs + 2 per merged occurrence (<= P0 in all) -> at most half full
    const uint64_t P0 = S - 2 * D;
    const uint64_t pcap = train_pow2(std::max<uint64_t>(6 * P0 + 1024, 1u << 12));
    if (pcap > (1ull << 32)) return fail(B200BPE_EINVAL, "corpus too large for one training call (pair table >= 2^32 slots)");
    CUDA_TRY(T.pkey.ensure(pcap)); CUDA_TRY(T.pcnt.ensure(pcap)); CUDA_TRY(T.pocc.ensure(pcap));
    CUDA_TRY(cudaMemsetAsync(T.pkey.p, 0xFF, pcap * 8, s)); CUDA_TRY(cudaMemsetAsync(T.pcnt.p, 0, pcap * 8, s));
    TrainPairs P{T.pkey.p, T.pcnt.p, T.pocc.p, pcap - 1};
    const uint64_t tcap = train_pow2(2ull * target + 1024);
    CUDA_TRY(T.th.ensure(target + 2)); CUDA_TRY(T.tpw.ensure(target + 2)); CUDA_TRY(T.tlen.ensure(target + 2));
    CUDA_TRY(T.tslot.ensure(tcap));
    CUDA_TRY(cudaMemsetAsync(T.tslot.p, 0xFF, tcap * 4, s));
    TrainTok TT{T.th.p, T.tpw.p, T.tlen.p, T.tslot.p, tcap - 1};
    train_tok_init_kernel<<<1, 32, 0, s>>>(TT);
    CUDA_TRY(T.stamp.ensure(D + 2)); CUDA_TRY(T.aff.ensure(D + 2)); CUDA_TRY(T.merges.ensure(3 * merges_cap + 3));
    CUDA_TRY(cudaMemsetAsync(T.stamp.p, 0, (D + 2) * 4, s));
    {
        TrainState init; memset(&init, 0, sizeof(init));
        init.best = ~0ull; init.n_ids = 256;
        *T.h_st = init;
        CUDA_TRY(cudaMemcpyAsync(T.st, T.h_st, sizeof(TrainState), cudaMemcpyHostToDevice, s));
    }
    if (D) train_pairs_init_kernel<<<n_sm * 8, 256, 0, s>>>(T.sym.p, T.woff.p, T.dlen.p, T.dcnt.p, D, P, T.st);
    CUDA_TRY(cudaEventRecord(T.ev[3], s));
    CUDA_TRY(cudaStreamSynchronize(s));
    CUDA_TRY(cudaGetLastError());
    ms_words += event_ms(T.ev[2], T.ev[3]);
    // ---- the merge loop: a CUDA graph of K steps, replayed until the state says stop ---------------------------------
    const int K = 128;
    const unsigned mark_grid = (unsigned)std::min<uint64_t>((S + 255) / 256 + 1, (uint64_t)n_sm * 16);
    CUDA_TRY(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    for (int k = 0; k < K; k++) {
        train_max_kernel<<<n_sm * 4, 256, 0, s>>>(P, T.st);
        train_first_kernel<<<n_sm * 4, 256, 0, s>>>(T.sym.p, S, P, T.st);
        train_commit_kernel<<<1, 32, 0, s>>>(T.sym.p, TT, T.merges.p, (uint32_t)merges_cap, target, T.st);
        train_mark_kernel<<<mark_grid, 256, 0, s>>>(T.sym.p, S, T.woff.p, D, T.stamp.p, T.aff.p, T.st);
        train_apply_kernel<<<n_sm * 8, 256, 0, s>>>(T.sym.p, T.woff.p, T.dlen.p, T.dcnt.p, T.aff.p, P, T.st);
    }
    {
        cudaError_t e = cudaStreamEndCapture(s, &T.graph);
        if (e != cudaSuccess) return fail(B200BPE_ECUDA, std::string("graph capture: ") + cudaGetErrorString(e));
    }
    CUDA_TRY(cudaGraphInstantiate(&T.exec, T.graph, 0));
    uint64_t batches = 0;
    CUDA_TRY(cudaEventRecord(T.ev[0], s));
    for (;;) {
        CUDA_TRY(cudaGraphLaunch(T.exec, s));
        batches++;
        CUDA_TRY(cudaMemcpyAsync(T.h_st, T.st, sizeof(TrainState), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        if (T.h_st->stop) break;
    }
    CUDA_TRY(cudaEventRecord(T.ev[1], s));
    CUDA_TRY(cudaStreamSynchronize(s));
    ms_loop = event_ms(T.ev[0], T.ev[1]);
    const TrainState fin = *T.h_st;
    if (fin.n_merges) CUDA_TRY(cudaMemcpy(merges_out, T.merges.p, (size_t)fin.n_merges * 12, cudaMemcpyDeviceToHost));
    *n_merges_out = fin.n_merges;
    if (stats8) {
        stats8[0] = (double)n_pieces; stats8[1] = (double)D; stats8[2] = (double)fin.n_merges; stats8[3] = (double)batches;
        stats8[4] = ms_split; stats8[5] = ms_words; stats8[6] = ms_loop; stats8[7] = (double)(cut.size() - 1);
    }
    if (fin.stop == TR_NOPAIR)
        return fail(B200BPE_ENOPAIR, "no pair left to merge: the corpus allows " + std::to_string(fin.n_ids) +
                                         " tokens, fewer than vocab_size = " + std::to_string(vocab_size));
    if (fin.stop == TR_CAP)
        return fail(B200BPE_ECAPACITY, "more than " + std::to_string(merges_cap) +
                                           " merges: too many merges produced bytes that already were a token");
    if (fin.stop != TR_DONE) return fail(B200BPE_ECUDA, "internal: training stopped with state " + std::to_string(fin.stop) +
                                                         ", error bits " + std::to_string(fin.err));
    return B200BPE_OK;
}
