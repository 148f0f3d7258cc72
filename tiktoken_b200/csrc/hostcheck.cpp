// hostcheck.cpp -- TEST-ONLY host build of the engine's __host__ __device__ building blocks.
// Compiled with plain g++ into libb200bpe_hostcheck.so and loaded only by tests (-m "not gpu"):
// it lets the CPU-only suite exercise exactly the rule / merge code the CUDA kernels execute.
// It is NOT part of libb200bpe.so and is never reachable from the product path.
#include <cstdint>
#include <cstring>
#include <vector>
#include "text_access.cuh"
#include "pretok_fast.cuh"
#include "unicode_classes.inc"

using namespace b2bpe;

extern "C" int hc_piece_starts(int pattern, const uint8_t *text, int64_t n, const uint64_t *doc_off,
                               int64_t n_docs, uint8_t *is_start /* n bytes, 0/1 */) {
    std::vector<uint8_t> padded((size_t)n + 8, 0);
    memcpy(padded.data(), text, (size_t)n);
    std::vector<uint32_t> dbits((size_t)(n + 63) / 32 + 1, 0);
    for (int64_t d = 0; d < n_docs; d++) {
        uint64_t o = doc_off[d];
        if ((int64_t)o < n) dbits[o >> 5] |= 1u << (o & 31);
    }
    uint8_t ascii[128];
    for (int i = 0; i < 128; i++) ascii[i] = UC_STAGE2[(uint32_t)UC_STAGE1[0] * 256 + i];
    TextAccess t{padded.data(), n, dbits.data(), UC_STAGE1, UC_STAGE2, ascii};
    for (int64_t pos = 0; pos < n; pos++) {
        uint8_t b = padded[pos];
        bool lead = (b & 0xC0u) != 0x80u;
        bool s;
        if (t.doc_start(pos)) s = true;
        else if (!lead) s = false;
        else if (pattern == PAT_R50K) s = boundary_before<PAT_R50K>(t, pos);
        else if (pattern == PAT_CL100K) s = boundary_before<PAT_CL100K>(t, pos);
        else if (pattern == PAT_O200K) s = boundary_before<PAT_O200K>(t, pos);
        else return -1;
        is_start[pos] = s ? 1 : 0;
    }
    return 0;
}

// ---- table build + per-thread short-piece path (piece probe, merge_short) --------------------
#include "bpe_tables.h"

struct HcTables { HostTables H; };

extern "C" void *hc_tables_new(const uint8_t *tok_bytes, const uint64_t *tok_off, const uint32_t *tok_rank,
                               uint32_t n, int *rc) {
    HcTables *h = new HcTables();
    *rc = build_tables(tok_bytes, tok_off, tok_rank, n, h->H);
    if (*rc) { delete h; return nullptr; }
    return h;
}
extern "C" void hc_tables_free(void *p) { delete (HcTables *)p; }
extern "C" uint64_t hc_tables_pairs(void *p) { return ((HcTables *)p)->H.n_pairs; }
// the two forms of the pair probe must agree: one at a time, two at a time
extern "C" uint32_t hc_pair_lookup(void *p, uint32_t a, uint32_t b) {
    DevTables T = ((HcTables *)p)->H.view();
    const uint32_t r = pair_lookup(T, a, b);
    uint32_t x, y; pair_lookup2(T, a, b, b, a, x, y);
    if (r != x || y != pair_lookup(T, b, a)) return 0xDEADBEEFu;
    return r;
}
// number of pair-table slots (one slot per probe step)
extern "C" uint64_t hc_pair_buckets(void *p) { return (uint64_t)((HcTables *)p)->H.pair_mask + 1; }
// whole-piece probe of 1..16 bytes (the probe kernel's issue / finish pair): rank or RANK_MAX
extern "C" uint32_t hc_piece_lookup(void *p, const uint8_t *piece, uint32_t len) {
    if (len == 0 || len > (uint32_t)SHORT_MAX) return 0xDEADBEEFu;
    uint64_t k0, k1; pack16(piece, len, k0, k1);
    return piece_lookup16(((HcTables *)p)->H.view(), k0, k1, len);
}
// the miss memo's key of a piece of 1..16 bytes, from the zero-padded words the probe kernel queues: 1 and the four key
// words, or 0 for a piece that is not memoised
extern "C" int hc_memo_key(const uint8_t *piece, uint32_t len, uint32_t *out4) {
    if (len == 0 || len > (uint32_t)SHORT_MAX) return -1;
    uint8_t b[16] = {0};
    memcpy(b, piece, len);
    U4 k; memcpy(&k, b, 16);
    if (!memo_key(k, len)) return 0;
    memcpy(out4, &k, 16);
    return 1;
}
// slots of the narrow and the wide piece table
extern "C" void hc_piece_slots(void *p, uint64_t *narrow, uint64_t *wide) {
    const HostTables &H = ((HcTables *)p)->H;
    *narrow = H.narrow_tab.size(); *wide = H.wide_tab.size() / 2;
}

// the short path of the encode kernel for one piece of 1..16 bytes: whole-piece probe
// (lib.rs:367-368) then merge_short; ids >= PSEUDO_BASE are reported as RANK_MAX.
extern "C" int hc_encode_short(void *p, const uint8_t *piece, uint32_t len, uint32_t *out) {
    const HostTables &H = ((HcTables *)p)->H;
    DevTables T = H.view();
    if (len == 0 || len > (uint32_t)SHORT_MAX) return -1;
    uint64_t k0, k1; pack16(piece, len, k0, k1);
    uint32_t r = piece_lookup16(T, k0, k1, len);
    if (r != RANK_MAX) { out[0] = r; return 1; }
    if (len == 1) { uint32_t id = T.byte_id[piece[0]]; out[0] = id >= PSEUDO_BASE ? RANK_MAX : id; return 1; }
    uint32_t id[32], rk[32], id2[32], rk2[32];
    uint32_t mask = merge_short(T, [&](int j) { return (uint32_t)piece[j]; }, (int)len, id, rk);
    // the warp-convergent variant the kernel uses must agree (n_max > n exercises the padding)
    uint32_t mask2 = merge_short_conv(T, [&](int j) { return (uint32_t)piece[j]; }, (int)len, SHORT_MAX, 1u, id2, rk2);
    if (mask2 != mask) return -2;
    for (uint32_t m = mask; m;) { int j = __builtin_ffs(m) - 1; m &= m - 1; if (id[j] != id2[j]) return -2; }
    int k = 0;
    for (uint32_t m = mask; m;) { int j = __builtin_ffs(m) - 1; m &= m - 1; out[k++] = id[j] >= PSEUDO_BASE ? RANK_MAX : id[j]; }
    return k;
}

// the thread-per-piece mid path (merge_mid_conv) for one piece of 2..cap bytes: whole-piece probe
// then merge; n_max > n exercises the padding.  ids >= PSEUDO_BASE are reported as RANK_MAX.
extern "C" int hc_encode_mid(void *p, const uint8_t *piece, uint32_t len, uint32_t cap, uint32_t *out) {
    const HostTables &H = ((HcTables *)p)->H;
    DevTables T = H.view();
    if (len < 2 || len > cap) return -1;
    uint32_t r = piece_lookup_long(T, long_hash_bytes(piece, len), len, [&](uint32_t i) { return piece[i]; });
    if (len <= (uint32_t)SHORT_MAX) { uint64_t k0, k1; pack16(piece, len, k0, k1); r = piece_lookup16(T, k0, k1, len); }
    if (r != RANK_MAX) { out[0] = r; return 1; }
    std::vector<uint32_t> id(cap + 8, 0xABABABABu), rk(cap + 8, 0xABABABABu), gmin(cap / MID_G + 2, 7u), gpos(cap / MID_G + 2, 7u);
    for (uint32_t j = 0; j < cap; j++) rk[j] = j < len ? piece[j] : 0u;          // the caller stages the bytes in rk
    merge_mid_conv(T, (int)len, (int)cap, 1u, id.data(), rk.data(), gmin.data(), gpos.data());
    int k = 0;
    for (uint32_t j = 0; j < len; j++) if (id[j] != ID_DEAD) out[k++] = id[j] >= PSEUDO_BASE ? RANK_MAX : id[j];
    return k;
}

// whole-piece probe for a long piece (> 16 bytes) through the hash + blob verification
extern "C" uint32_t hc_probe_long(void *p, const uint8_t *piece, uint32_t len) {
    const HostTables &H = ((HcTables *)p)->H;
    DevTables T = H.view();
    uint64_t h = long_hash_bytes(piece, len);
    return piece_lookup_long(T, h, len, [&](uint32_t i) { return piece[i]; });
}

// the bit-parallel span evaluator the pre-tokeniser kernel actually runs (pretok_fast.cuh)
template <bool CUT>
static int piece_starts_fast(int pattern, const uint8_t *text, int64_t n, const uint64_t *doc_off, int64_t n_docs,
                             uint8_t *is_start, uint64_t *stats2) {
    std::vector<uint8_t> padded((size_t)n + 64, 0);
    memcpy(padded.data(), text, (size_t)n);
    const int64_t n_words = (n + 1 + 31) / 32;
    std::vector<uint32_t> dbits((size_t)n_words + 4, 0);
    for (int64_t d = 0; d <= n_docs; d++) {
        uint64_t o = doc_off[d];
        dbits[o >> 5] |= 1u << (o & 31);
    }
    uint8_t ascii[128];
    for (int i = 0; i < 128; i++) ascii[i] = UC_STAGE2[(uint32_t)UC_STAGE1[0] * 256 + i];
    TextAccess t{padded.data(), n, dbits.data(), UC_STAGE1, UC_STAGE2, ascii};
    SpanStats st{0, 0};
    for (int64_t w = 0; w < n_words; w++) {
        uint32_t word;
        if (pattern == PAT_R50K) word = span_boundaries<PAT_R50K, CUT>(t, w, &st);
        else if (pattern == PAT_CL100K) word = span_boundaries<PAT_CL100K, CUT>(t, w, &st);
        else if (pattern == PAT_O200K) word = span_boundaries<PAT_O200K, CUT>(t, w, &st);
        else return -1;
        for (int j = 0; j < 32; j++) {
            int64_t pos = w * 32 + j;
            if (pos <= n) is_start[pos] = (word >> j) & 1u;
        }
    }
    if (stats2) { stats2[0] = st.positions; stats2[1] = st.slow; }
    return 0;
}
extern "C" int hc_piece_starts_fast(int pattern, const uint8_t *text, int64_t n, const uint64_t *doc_off,
                                    int64_t n_docs, uint8_t *is_start /* n+1 bytes */, uint64_t *stats2) {
    return piece_starts_fast<false>(pattern, text, n, doc_off, n_docs, is_start, stats2);
}
// the same, as the bytes mode's pre-tokeniser runs it (pretok_kernel<PAT, true>): haystack starts may follow ill-formed leads
extern "C" int hc_piece_starts_fast_cut(int pattern, const uint8_t *text, int64_t n, const uint64_t *doc_off,
                                        int64_t n_docs, uint8_t *is_start, uint64_t *stats2) {
    return piece_starts_fast<true>(pattern, text, n, doc_off, n_docs, is_start, stats2);
}

// the host path's seam rule and chunk plan (doc_seams.h), as b200bpe.cu runs them
#include "doc_seams.h"

extern "C" int hc_is_seam(const uint8_t *text, uint64_t doc_lo, uint64_t doc_hi, uint64_t p) {
    return is_seam(text, doc_lo, doc_hi, p) ? 1 : 0;
}
// specials: sp_n strings, string i = sp_bytes[sp_off[i] .. sp_off[i+1]); flags NULL: no special handling.  Returns the
// number of chunks n (or -1 - PlanError); when n <= cap: bounds[0..n] = the chunks' byte bounds, first_doc[0..n] and
// head[0..n-1] as in ChunkPlan; stats2 = {seams, docs_cut}.
extern "C" int64_t hc_plan_chunks(const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs, uint64_t chunk, int mode,
                                  const uint8_t *sp_bytes, const uint64_t *sp_off, uint64_t sp_n, const uint8_t *flags,
                                  uint64_t cap, uint64_t *bounds, uint64_t *first_doc, uint8_t *head, uint64_t *stats2) {
    std::vector<std::string> specials;
    for (uint64_t i = 0; i < sp_n; i++) specials.emplace_back((const char *)sp_bytes + sp_off[i], (size_t)(sp_off[i + 1] - sp_off[i]));
    SeamSpecials sp;
    sp.str = specials.data(); sp.n = specials.size(); sp.flags = flags;
    ChunkPlan P;
    const int rc = plan_chunks(text, doc_off, n_docs, chunk, (PlanMode)mode, sp, P);
    if (rc) return -1 - rc;
    const uint64_t n = P.cut.size() - 1;
    const uint64_t *po = P.part_off.empty() ? doc_off : P.part_off.data();
    if (n <= cap) {
        for (uint64_t c = 0; c <= n; c++) { bounds[c] = po[P.cut[c]]; first_doc[c] = P.first_doc[c]; }
        for (uint64_t c = 0; c < n; c++) head[c] = P.head[c];
    }
    stats2[0] = P.seams; stats2[1] = P.docs_cut;
    return (int64_t)n;
}

// the UTF-8 classifier of the bytes mode (utf8_check.cuh): valid_up_to of every document (its length when well-formed),
// from the first mark of each document, the way utf8_check_kernel reduces them
#include "utf8_check.cuh"

extern "C" int hc_utf8_valid_up_to(const uint8_t *text, int64_t n, const uint64_t *doc_off, int64_t n_docs, uint64_t *vup) {
    const int64_t n_words = (n + 1 + 31) / 32;
    std::vector<uint32_t> dbits((size_t)n_words + 4, 0);
    for (int64_t d = 0; d <= n_docs; d++) dbits[doc_off[d] >> 5] |= 1u << (doc_off[d] & 31);
    for (int64_t d = 0; d < n_docs; d++) vup[d] = doc_off[d + 1] - doc_off[d];
    int64_t d = 0;
    for (int64_t w = 0; w < n_words; w++) {
        for (uint32_t m = utf8_bad_word(text, n, dbits.data(), w); m; m &= m - 1) {
            const uint64_t pos = (uint64_t)(w * 32 + __builtin_ctz(m));
            while (doc_off[d + 1] <= pos) d++;
            if (pos - doc_off[d] < vup[d]) vup[d] = pos - doc_off[d];
        }
    }
    return 0;
}
