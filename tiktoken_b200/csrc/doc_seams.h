// doc_seams.h -- the host path's chunk plan: where a batch may be cut into chunks, inside documents included.
// Plain C++ (no CUDA): b200bpe.cu plans with it and hostcheck.cpp exposes it to the CPU tests.
//
// A document may be cut at a position p (a "seam") only where the split into pieces provably does not depend on the
// cut: split(text) == split(text[:p]) + split(text[p:]).  BPE runs per piece, so the tokens of the parts, back to back,
// are then those of the whole document.  None of the three patterns has a lookbehind, so a piece that starts at p
// matches the same way with or without the text before p; the two rules below also make sure that the piece before p
// ends at p with or without the text after it.  Both look at ASCII bytes only (DESIGN.md "Seams"):
//   R1 (word gap)   text[p-1] is an ASCII letter, text[p] == ' ', text[p+1] is an ASCII letter;
//   R2 (line start) text[p-2] is in 0x21..0x7E, text[p-1] == '\n', text[p] is an ASCII letter or digit.
#pragma once
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

namespace b2bpe {

inline bool seam_letter(uint8_t c) { return (uint8_t)((c | 0x20) - 'a') < 26; }
inline bool seam_digit(uint8_t c) { return (uint8_t)(c - '0') < 10; }

// R1 or R2 at p of the document [doc_lo, doc_hi); false unless p lies strictly inside it with the bytes the rule reads
inline bool is_seam(const uint8_t *text, uint64_t doc_lo, uint64_t doc_hi, uint64_t p) {
    if (p <= doc_lo || p >= doc_hi) return false;
    const uint8_t a = text[p - 1], b = text[p];
    if (b == ' ') return p + 1 < doc_hi && seam_letter(a) && seam_letter(text[p + 1]);
    return a == '\n' && p >= doc_lo + 2 && (uint8_t)(text[p - 2] - 0x21) < 0x5E && (seam_letter(b) || seam_digit(b));
}

// The special tokens of a call: a seam must not fall inside an occurrence of a special the call allows or disallows
// (flags[i] != 0), so that every occurrence lies in one part: allowed ones cut the same haystacks, and the leftmost
// disallowed one is still found.  flags == NULL: the call has no special handling.
struct SeamSpecials {
    const std::string *str = nullptr; size_t n = 0; const uint8_t *flags = nullptr;
};

inline bool straddles_special(const uint8_t *text, uint64_t doc_lo, uint64_t doc_hi, uint64_t p, const SeamSpecials &sp) {
    if (!sp.flags) return false;
    for (size_t i = 0; i < sp.n; i++) {
        const uint64_t len = sp.str[i].size();
        if (!sp.flags[i] || len < 2) continue;
        for (uint64_t q = p - std::min<uint64_t>(len - 1, p - doc_lo); q < p && q + len <= doc_hi; q++)
            if (memcmp(text + q, sp.str[i].data(), (size_t)len) == 0) return true;
    }
    return false;
}

inline bool usable_seam(const uint8_t *text, uint64_t doc_lo, uint64_t doc_hi, uint64_t p, const SeamSpecials &sp) {
    return is_seam(text, doc_lo, doc_hi, p) && !straddles_special(text, doc_lo, doc_hi, p, sp);
}

// The seam for target t in the document [doc_lo, doc_hi), for a chunk that starts at pos: the last one in
// [t - win, t], else the first one in (t, t + win]; always > pos.  0 when there is none.
inline uint64_t find_seam(const uint8_t *text, uint64_t doc_lo, uint64_t doc_hi, uint64_t pos, uint64_t t, uint64_t win,
                          const SeamSpecials &sp) {
    const uint64_t lo = std::max(pos + 1, t > win ? t - win : 0);
    for (uint64_t p = std::min(t, doc_hi); p >= lo && p > 0; p--)
        if (usable_seam(text, doc_lo, doc_hi, p, sp)) return p;
    for (uint64_t p = std::max(t + 1, lo); p <= t + win && p < doc_hi; p++)
        if (usable_seam(text, doc_lo, doc_hi, p, sp)) return p;
    return 0;
}

enum PlanMode { PLAN_WHOLE = 0, PLAN_DOCS = 1, PLAN_SEAMS = 2 };
enum PlanError { PLAN_OK = 0, PLAN_UNORDERED = 1, PLAN_TOO_LARGE = 2 };
static const uint64_t PLAN_MAX_CHUNK = (1ull << 32) - 4096;     // bytes of one pipeline run

// The pipeline runs on parts: documents, or the pieces of a document between its seams.
struct ChunkPlan {
    std::vector<uint64_t> part_off;   // byte offsets of the parts when some document was cut; empty: the parts are the documents
    std::vector<uint64_t> cut;        // chunk c = parts [cut[c], cut[c+1])
    std::vector<uint64_t> first_doc;  // chunk c holds the starts of documents [first_doc[c], first_doc[c+1])
    std::vector<uint8_t> head;        // chunk c starts at a seam: 1, or 2 when that is its document's first seam; else 0
    uint64_t seams = 0, docs_cut = 0;
};

// Chunks of about `chunk` bytes; one chunk when the batch is at most 1.5 chunks or mode is PLAN_WHOLE.  A chunk ends
// at the last document boundary within `chunk` bytes of its start.  A document larger than that is a chunk of its own
// under PLAN_DOCS, and under PLAN_SEAMS when it is at most two chunks long (a cut would leave a small rest for little
// overlap).  A longer one is cut at the seam find_seam picks for the target `chunk` bytes after the chunk's start
// (window chunk / 4), or, when there is none, for the target a chunk later, and so on; the chunk after a seam starts
// with the rest of the document.  Batches whose documents are all at most two chunks long, and documents without a
// seam, plan exactly as under PLAN_DOCS.  A pure function of its arguments.
inline int plan_chunks(const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs, uint64_t chunk, PlanMode mode,
                       const SeamSpecials &sp, ChunkPlan &P) {
    const uint64_t n_bytes = doc_off[n_docs];
    P = ChunkPlan();
    std::vector<uint64_t> b(1, 0);    // chunk c = bytes [b[c], b[c+1])
    P.first_doc.assign(1, 0);
    P.head.clear();
    if (mode != PLAN_WHOLE && n_bytes > chunk + chunk / 2) {
        const uint64_t win = chunk / 4;
        uint64_t lo = 0, pos = 0;     // the next document to start, the byte the next chunk starts at
        uint8_t head = 0;             // pos is a seam inside document lo - 1 (1), its first one (2)
        while (lo < n_docs || head) {
            const uint64_t want = pos + chunk, first = head ? lo : lo + 1;
            const uint64_t k = (uint64_t)(std::upper_bound(doc_off + first, doc_off + n_docs + 1, want) - doc_off);
            uint64_t end, next_lo;
            bool seam = false;
            if (k > first) { next_lo = k - 1; end = doc_off[next_lo]; }   // the last document boundary <= want
            else {                                                        // document d is larger than the rest of the chunk
                const uint64_t d = first - 1, dlo = doc_off[d], dhi = doc_off[d + 1];
                next_lo = d + 1; end = dhi;
                if (mode == PLAN_SEAMS && dlo <= pos && pos < dhi && dhi <= n_bytes && dhi - dlo > 2 * chunk)
                    for (uint64_t t = want; t < dhi; t += chunk)
                        if (uint64_t p = find_seam(text, dlo, dhi, pos, t, win, sp)) { end = p; next_lo = head ? lo : lo + 1; seam = true; break; }
            }
            P.head.push_back(head);
            b.push_back(end); P.first_doc.push_back(next_lo);
            if (seam) { P.seams++; P.docs_cut += head ? 0 : 1; }
            head = seam ? (head ? 1 : 2) : 0;
            lo = next_lo; pos = end;
        }
    } else {
        b.push_back(n_bytes); P.first_doc.push_back(n_docs); P.head.push_back(0);
    }
    for (size_t c = 0; c + 1 < b.size(); c++) {
        if (b[c + 1] < b[c]) return PLAN_UNORDERED;
        if (b[c + 1] - b[c] >= PLAN_MAX_CHUNK) return PLAN_TOO_LARGE;
    }
    if (!P.seams) { P.cut = P.first_doc; return PLAN_OK; }
    // parts: every chunk's seam (its first byte) and the starts of its documents, then the end of the batch
    const size_t n_chunks = b.size() - 1;
    P.part_off.reserve((size_t)n_docs + (size_t)P.seams + 1);
    for (size_t c = 0; c < n_chunks; c++) {
        P.cut.push_back(P.part_off.size());
        if (P.head[c]) P.part_off.push_back(b[c]);
        for (uint64_t d = P.first_doc[c]; d < P.first_doc[c + 1]; d++) P.part_off.push_back(doc_off[d]);
    }
    P.cut.push_back(P.part_off.size());
    P.part_off.push_back(n_bytes);
    return PLAN_OK;
}

}  // namespace b2bpe
