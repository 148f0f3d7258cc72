// pretok_fast.cuh -- bit-parallel evaluation of the pre-tokeniser rules for one 32-byte span.
//
// pretok_rules.cuh decides each position on its own with ~100-200 instructions.  Here a thread
// classifies a 48-byte window (its 32 bytes, 8 before, 8 after) with SWAR byte tests, gathers
// the classes into 64-bit masks (bit i = byte i of the window, multi-byte scalars carry their
// class on every byte) and evaluates the rules for all 32 positions at once with shifts and
// logic ops.  Every position whose outcome is not fully determined by that local picture
// (contractions, digit runs of 3+, CR/LF look-ahead, o200k case/mark subtleties, multi-byte
// neighbours, ...) is flagged `slow` and decided by the general, proven rule function
// boundary_before<PAT>().  So the fast path never has to be complete, only right where it
// claims to be; tests/test_pretok_rules.py checks it exhaustively against the oracle.
#pragma once
#include "text_access.cuh"

namespace b2bpe {

struct SpanStats { unsigned long long positions, slow; };


#if defined(__CUDA_ARCH__)
#define B2_CTZLL(x) (__ffsll((long long)(x)) - 1)
#define B2_POPCLL(x) __popcll(x)
#else
#define B2_CTZLL(x) __builtin_ctzll(x)
#define B2_POPCLL(x) __builtin_popcountll(x)
#endif

// ---- SWAR classification of the 48-byte window ------------------------------------------------------------------
// The window's bytes are first TRANSPOSED with byte permutes (PRMT): own word T[k] holds the own bytes {k, 8+k, 16+k,
// 24+k}, halo word H[k] the halo bytes {k, 4+k | 40+k, 44+k}.  A per-byte test leaves its answer in bit 7 of every byte
// (other bits: don't care, all combining logic is bitwise); with the transposed layout the 32 answers of a class fall
// into place with ONE shift-and-or per word -- acc |= f >> (7-k) puts byte 8j+k at bit 8j+k -- instead of a
// multiply-gather and a 64-bit insert per word and class.
B2_HD uint32_t b2_prmt(uint32_t a, uint32_t b, uint32_t sel) {
#if defined(__CUDA_ARCH__)
    return __byte_perm(a, b, sel);
#else
    const uint64_t v = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((v >> (8 * ((sel >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
    return r;
#endif
}
// 4 x 4 byte transpose: t[k] = { a.byte k, b.byte k, c.byte k, d.byte k }
B2_HD void transpose4(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t &t0, uint32_t &t1, uint32_t &t2, uint32_t &t3) {
    const uint32_t ab_lo = b2_prmt(a, b, 0x5140u), ab_hi = b2_prmt(a, b, 0x7362u);
    const uint32_t cd_lo = b2_prmt(c, d, 0x5140u), cd_hi = b2_prmt(c, d, 0x7362u);
    t0 = b2_prmt(ab_lo, cd_lo, 0x5410u); t1 = b2_prmt(ab_lo, cd_lo, 0x7632u);
    t2 = b2_prmt(ab_hi, cd_hi, 0x5410u); t3 = b2_prmt(ab_hi, cd_hi, 0x7632u);
}

struct ClassAcc {             // bit (8j + k) of every member = the answer for byte lane j of transposed word k
    uint32_t hi, cont, al, up, dg, sp, ws, nl, ap, sl;
};
B2_HD uint32_t b2_mad1(uint32_t v, uint32_t one, uint32_t c) {   // v * one + c as ONE multiply-add (no common `v * one`)
#if defined(__CUDA_ARCH__)
    uint32_t r;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(v), "r"(one), "r"(c));
    return r;
#else
    return v * one + c;
#endif
}
// The byte tests of one (transposed) word.  Pipe balance matters more than the instruction count here: the kernel is
// bound by the ALU pipe (LOP3 / SHF / IADD3: one warp instruction per two cycles and scheduler) while the FMA pipe,
// which executes IMAD, idles.  So the 15 per-byte comparisons of a word are written as multiply-adds
// (v * one + c with `one` == 1 at run time, opaque to the compiler -> IMAD); the combining logic and the accumulation
// (one LEA.HI / SHF+LOP3 per class) stay on the ALU pipe.  A multiply-high accumulate (IMAD.HI) would
// move more work off the ALU pipe, but IMAD.HI issues at a quarter of the IMAD rate.
template <int K>
B2_HD void classify_word(uint32_t x, ClassAcc &a, uint32_t one) {
    const uint32_t y = x & 0x7F7F7F7Fu, yl = y | 0x20202020u;
    const uint32_t hi7 = x & 0x80808080u, nx7 = hi7 ^ 0x80808080u;       // bit 7 of every byte: non-ASCII / ASCII
#define B2_GE(v, n) b2_mad1(v, one, (0x80u - (uint32_t)(n)) * 0x01010101u)  /* bit 7 of every byte: (7-bit v) >= n */
    const uint32_t alpha = B2_GE(yl, 'a') & ~B2_GE(yl, 'z' + 1) & nx7;
    const uint32_t upper = alpha & ~(x << 2);                              // bit 5 clear
    const uint32_t digit = B2_GE(y, '0') & ~B2_GE(y, '9' + 1) & nx7;
    const uint32_t space = B2_GE(y, 0x20) & ~B2_GE(y, 0x21) & nx7;
    const uint32_t g0e = B2_GE(y, 0x0E);
    const uint32_t nl_a = B2_GE(y, 0x0A) & ~B2_GE(y, 0x0B) & nx7, nl_d = B2_GE(y, 0x0D) & ~g0e & nx7;
    const uint32_t ws5 = B2_GE(y, 0x09) & ~g0e & nx7;                      // 0x09..0x0D; CR / LF are taken out on the masks
    const uint32_t apos = B2_GE(y, 0x27) & ~B2_GE(y, 0x28) & nx7;
    const uint32_t slash = B2_GE(y, 0x2F) & ~B2_GE(y, 0x30) & nx7;
    const uint32_t cnt = hi7 & ~(x << 1);                                  // 10xxxxxx
#undef B2_GE
#define B2_ACC(dst, f) dst |= (f) >> (7 - K)                               /* the answers are masked to bit 7 of every byte */
    B2_ACC(a.hi, hi7); B2_ACC(a.cont, cnt); B2_ACC(a.al, alpha); B2_ACC(a.up, upper); B2_ACC(a.dg, digit);
    B2_ACC(a.sp, space); B2_ACC(a.ws, ws5); B2_ACC(a.nl, nl_a); B2_ACC(a.nl, nl_d); B2_ACC(a.ap, apos); B2_ACC(a.sl, slash);
#undef B2_ACC
}

// own answers (bit i = own byte i) and halo answers (nibbles at bits 0, 8 | 16, 24) -> window mask (bit i = window byte i)
B2_HD uint64_t window_mask(uint32_t own, uint32_t halo) {
    const uint32_t pre = (halo & 0xFu) | ((halo >> 4) & 0xF0u);
    const uint32_t post = ((halo >> 16) & 0xFu) | ((halo >> 20) & 0xF0u);
    return (uint64_t)pre | ((uint64_t)own << 8) | ((uint64_t)post << 40);
}

struct WinMasks {
    uint64_t valid, D, hi, cont;
    uint64_t LU, LL, LB, M, N, NA, SP, WS, NL, APOS, SLASH, O;   // WS: non-SP non-CR/LF whitespace
};

// Classify the window [win0, win0+48).  Non-ASCII scalars are decoded one by one.  CUT (bytes mode, where a document
// may end in an ill-formed lead byte): a lead does not paint its class past the next document or haystack start.
template <bool CUT = false>
B2_HD void classify_window(const TextAccess &t, int64_t win0, int64_t w, WinMasks &m) {
    uint32_t W[12];
    const int64_t n = t.n;
#if defined(__CUDA_ARCH__)
    if (win0 >= 0 && win0 + 48 <= (n & ~7ll)) {
        const uint2 *p = reinterpret_cast<const uint2 *>(t.text + win0);
#pragma unroll
        for (int k = 0; k < 6; k++) { uint2 v = __ldg(p + k); W[2 * k] = v.x; W[2 * k + 1] = v.y; }
    } else
#endif
    {
        for (int k = 0; k < 12; k++) {
            uint32_t x = 0;
            for (int b = 0; b < 4; b++) {
                int64_t pos = win0 + 4 * k + b;
                if (pos >= 0 && pos < n) x |= (uint32_t)t.text[pos] << (8 * b);
            }
            W[k] = x;
        }
    }
    uint64_t valid = 0xFFFFFFFFFFFFull;
    if (win0 < 0) valid &= ~((1ull << (-win0)) - 1ull);
    if (win0 + 48 > n) { int64_t keep = n - win0; valid &= keep <= 0 ? 0ull : ((1ull << keep) - 1ull); }
    uint32_t T[8], H[4];
    transpose4(W[2], W[4], W[6], W[8], T[0], T[1], T[2], T[3]);          // own bytes 8j + k      (k = 0..3)
    transpose4(W[3], W[5], W[7], W[9], T[4], T[5], T[6], T[7]);          //                        (k = 4..7)
    transpose4(W[0], W[1], W[10], W[11], H[0], H[1], H[2], H[3]);        // halo: window bytes k, 4+k | 40+k, 44+k
    ClassAcc o = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}, h = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    const uint32_t one = t.one;
    classify_word<0>(T[0], o, one); classify_word<1>(T[1], o, one); classify_word<2>(T[2], o, one); classify_word<3>(T[3], o, one);
    classify_word<4>(T[4], o, one); classify_word<5>(T[5], o, one); classify_word<6>(T[6], o, one); classify_word<7>(T[7], o, one);
    classify_word<0>(H[0], h, one); classify_word<1>(H[1], h, one); classify_word<2>(H[2], h, one); classify_word<3>(H[3], h, one);
    const uint64_t hi = window_mask(o.hi, h.hi), cont = window_mask(o.cont, h.cont), al = window_mask(o.al, h.al);
    const uint64_t up = window_mask(o.up, h.up), dg = window_mask(o.dg, h.dg), sp = window_mask(o.sp, h.sp);
    const uint64_t nl = window_mask(o.nl, h.nl), ws = window_mask(o.ws, h.ws) & ~nl, ap = window_mask(o.ap, h.ap);
    const uint64_t sl = window_mask(o.sl, h.sl);
    m.valid = valid; m.hi = hi & valid; m.cont = cont & valid;
    m.LU = up & valid; m.LL = (al & ~up) & valid; m.LB = 0; m.M = 0;
    m.N = dg & valid; m.NA = m.N; m.SP = sp & valid; m.WS = ws & valid; m.NL = nl & valid;
    m.APOS = ap & valid; m.SLASH = sl & valid;
    uint64_t ascii_known = m.LU | m.LL | m.N | m.SP | m.WS | m.NL | m.APOS | m.SLASH;
    m.O = valid & ~m.hi & ~ascii_known;
    // doc-start bits of the window: words w-1 (top byte), w, w+1 (low byte)
    uint64_t D = (uint64_t)t.dbits[w] << 8;
    if (w > 0) D |= (uint64_t)(t.dbits[w - 1] >> 24);
    D |= (uint64_t)(t.dbits[w + 1] & 0xFFu) << 40;
    m.D = D & valid;
    // non-ASCII scalars: decode, look up, paint the class on all their bytes
    for (uint64_t leads = m.hi & ~m.cont; leads;) {
        const int j = B2_CTZLL(leads); leads &= leads - 1;
        const int64_t pos = win0 + j;
        const unsigned b = t.text[pos];
        const int len = b < 0xE0 ? 2 : b < 0xF0 ? 3 : 4;
        if (pos + len > n) continue;                 // truncated tail: stays "unknown", handled by slow path
        const int c = t.cls(pos);
        uint64_t bits = ((1ull << len) - 1ull) << j;
        bits &= valid;
        if (CUT) {
            const uint64_t cross = D & bits & ~(1ull << j);
            if (cross) bits &= (cross & (0ull - cross)) - 1ull;
        }
        switch (c) {
            case C_LU: m.LU |= bits; break;
            case C_LL: m.LL |= bits; break;
            case C_LB: m.LB |= bits; break;
            case C_M: m.M |= bits; break;
            case C_N: m.N |= bits; break;
            case C_WS: m.WS |= bits; break;
            default: m.O |= bits; break;
        }
    }
}

// Fast part of a span: returns the boundary bits the local picture decides (window bit i = byte win0 + i,
// own bytes are bits 8..39; document starts included) and, in `slow_out`, the own positions that
// must be decided by the general rule function boundary_before<PAT>().
template <int PAT, bool CUT = false>
B2_HD uint64_t span_fast(const TextAccess &t, int64_t w, uint64_t &slow_out, SpanStats *stats = nullptr) {
    const int64_t base = w * 32, win0 = base - 8;
    slow_out = 0;
    if (base > t.n) return 0;
    WinMasks m;
    classify_window<CUT>(t, win0, w, m);
    const uint64_t OWN = 0xFFFFFFFFull << 8;
    const uint64_t lead = m.valid & ~m.cont;
    const uint64_t own = OWN & lead & ~m.D;              // positions to decide (doc starts are forced)
    const uint64_t L = m.LU | m.LL | m.LB;
    const uint64_t WSnn = m.SP | m.WS;                   // whitespace that is not CR/LF
    const uint64_t WSany = WSnn | m.NL;
    const uint64_t aposNear = (m.APOS << 2) | (m.APOS << 3);
    // "next scalar exists in this document and is not whitespace", for single-byte current scalars
    const uint64_t nextNonWs = ((m.valid & ~m.D & ~WSany) >> 1);
    const uint64_t pL = L << 1, pN = m.N << 1, pSP = m.SP << 1, pNL = m.NL << 1, pWSnn = WSnn << 1;
    const uint64_t pWSany = WSany << 1, pAPOS = m.APOS << 1, pHi = m.hi << 1;
    uint64_t b = 0, slow = 0;
    const uint64_t unk0 = m.valid & ~(m.LU | m.LL | m.LB | m.M | m.N | m.SP | m.WS | m.NL | m.APOS | m.SLASH | m.O);
    if (PAT == PAT_R50K) {
        const uint64_t X = m.O | m.APOS | m.SLASH | m.M;
        const uint64_t pX = X << 1;
        b |= WSany & (~pWSany | nextNonWs);
        slow |= WSany & m.hi & pWSany;
        b |= L & ~(pL | pSP);
        slow |= L & (pAPOS | (pL & aposNear));
        b |= m.N & ~(pN | pSP);
        b |= X & ~(pX | pSP);
    } else if (PAT == PAT_CL100K) {
        const uint64_t X = m.O | m.APOS | m.SLASH | m.M;
        const uint64_t pX = X << 1;
        // letters
        b |= L & (pN | pNL);
        b |= L & pX & ~pHi & ~(m.D << 1) & ((X | m.SP) << 2);
        // Letters next to an apostrophe a (the only undecided positions of English text).  The letter at a+1 needs
        // nothing special: whether a starts `'s` or is the one-scalar prefix of a word, no piece starts at a+1
        // when one starts at a, and the rule above covers an apostrophe inside a punctuation run.  The letters at
        // a+2 / a+3 (behind letters) are where the first alternative `'(?i:[sdmt]|ll|ve|re)` may have ended:
        //   boundary(a+2) = starts(a) & [sdmt](a+1);   boundary(a+3) = starts(a) & ![sdmt](a+1) & (ll|ve|re)(a+1,a+2)
        // decided per apostrophe with two byte loads (apostrophes are sparse).  Non-ASCII letters in the suffix
        // position (U+017F folds to s) stay with the general function.
        slow |= L & (pX & pHi);
        {
            const uint64_t starts = m.APOS & (~(pX | pSP) | m.D);
            const uint64_t cand = L & pL & aposNear & own;
            uint64_t und = cand;
            for (uint64_t aps = m.APOS & ((cand >> 2) | (cand >> 3)); aps;) {
                const int j = B2_CTZLL(aps); aps &= aps - 1;
                const uint64_t a1 = 1ull << (j + 1), a2 = a1 << 1, a3 = a2 << 1;
                if (!(L & a1) || (m.hi & a1)) continue;                       // a+1 is not an ASCII letter
                const bool st = (starts >> j) & 1ull;
                const unsigned c1 = t.text[win0 + j + 1] | 0x20u;
                const bool sdmt = c1 == 's' || c1 == 'd' || c1 == 'm' || c1 == 't';
                if (cand & a2) {
                    if (!(m.D & a1) && st && sdmt) b |= a2;
                    und &= ~a2;
                }
                if ((cand & a3) && !(m.hi & a2)) {                              // a+2 is an ASCII letter (cand: letter before a+3)
                    const unsigned c2 = t.text[win0 + j + 2] | 0x20u;
                    const bool two = (c1 == 'l' && c2 == 'l') || (c1 == 'v' && c2 == 'e') || (c1 == 'r' && c2 == 'e');
                    if (!(m.D & (a1 | a2)) && st && !sdmt && two) b |= a3;
                    und &= ~a3;
                }
            }
            slow |= und;
        }
        // digits: groups of three from the run start
        b |= m.N & ~pN;
        {   // `\p{N}{1,3}`: a digit starts a piece iff the count of digits before it in its run is a
            // multiple of 3.  Runs of ASCII digits that start within the 8-byte look-back are counted with
            // shifts; longer or non-ASCII runs go the slow way.
            const uint64_t A = m.NA;
            // an ASCII digit that starts its run.  A byte whose class is unknown here (continuation bytes of a
            // scalar that begins before the window) may belong to a non-ASCII digit: no known run start after it
            const uint64_t rs = A & ~((m.N | unk0) << 1);
            const uint64_t c1 = A << 1, c2 = c1 & (A << 2), c3 = c2 & (A << 3), c4 = c3 & (A << 4);
            const uint64_t c5 = c4 & (A << 5), c6 = c5 & (A << 6), c7 = c6 & (A << 7);
            const uint64_t k1 = rs << 1, k2 = c1 & (rs << 2), k3 = c2 & (rs << 3), k4 = c3 & (rs << 4);
            const uint64_t k5 = c4 & (rs << 5), k6 = c5 & (rs << 6), k7 = c6 & (rs << 7);
            const uint64_t known = (k1 | k2 | k3 | k4 | k5 | k6 | k7) & ~(m.D | (m.D << 1) | (m.D << 2) | (m.D << 3) |
                                   (m.D << 4) | (m.D << 5) | (m.D << 6));
            (void)c7;
            b |= A & pN & known & (k3 | k6);
            slow |= m.N & pN & ~(A & known);
        }
        b |= X & ~(pX | pSP);
        b |= m.NL & (pL | pN);
        b |= WSnn & ~pWSany;
        b |= WSnn & pWSnn & nextNonWs;
        slow |= WSnn & (pNL | (m.hi & pWSany));
    } else {
        const uint64_t Xo = m.O | m.APOS | m.SLASH;
        const uint64_t pM = m.M << 1, pLB = m.LB << 1, pLL = m.LL << 1, pLU = m.LU << 1;
        const uint64_t low = m.LL | m.LB;                           // extends any word
        b |= low & (pN | pNL);
        b |= m.LU & (pLL | pN | pNL);
        // A letter right after an "other" scalar x (punctuation, symbol; not apostrophe / slash / mark): x is either
        // the optional one-scalar prefix of the word (a piece starts AT x) or the end of a punctuation run (a piece
        // started before x), so  boundary(p) = !boundary(x),  and boundary(x) follows from the scalar before x:
        // letter / digit / non-space whitespace / CR-LF / document start => a piece starts at x;  space, other or
        // apostrophe => x continues (or is joined to) what precedes it.  x may be 1..4 bytes long.
        {
            const uint64_t pO = m.O << 1, leadNA = m.hi & ~m.cont, c1 = m.cont << 1, c2 = m.cont << 2, c3 = m.cont << 3;
            const uint64_t len1 = pO & ~(m.hi << 1), len2 = pO & c1 & (leadNA << 2), len3 = pO & c1 & c2 & (leadNA << 3);
            const uint64_t len4 = pO & c1 & c2 & c3 & (leadNA << 4);
            const uint64_t Q1 = L | m.N | m.WS | m.NL, Q0 = m.SP | m.O | m.APOS;
            const uint64_t atD = (len1 & (m.D << 1)) | (len2 & (m.D << 2)) | (len3 & (m.D << 3)) | (len4 & (m.D << 4));
            const uint64_t x1 = (len1 & (Q1 << 2)) | (len2 & (Q1 << 3)) | (len3 & (Q1 << 4)) | (len4 & (Q1 << 5)) | atD;
            const uint64_t x0 = ((len1 & (Q0 << 2)) | (len2 & (Q0 << 3)) | (len3 & (Q0 << 4)) | (len4 & (Q0 << 5))) & ~atD;
            const uint64_t letter_after_o = (low | m.LU) & pO;
            b |= letter_after_o & x0;
            slow |= letter_after_o & ~(x0 | x1);
            // Apostrophes, and the letters up to three bytes behind one, decided per apostrophe (they are sparse):
            //  * after a word character, `'s|'t|'re|'ve|'m|'ll|'d` (ASCII, any case) is the optional tail of that word's
            //    piece: no piece starts at the apostrophe or inside the suffix, one starts right after it; anything else
            //    makes the apostrophe an ordinary "other" scalar that starts a piece and prefixes the letters after it;
            //  * after anything else it is an ordinary "other" scalar: boundary from the scalar before it, and the letter
            //    after it gets the opposite (prefix rule above).
            // Chains ('s'd: an apostrophe 2-3 bytes behind another), marks, slashes and non-ASCII suffix letters (U+017F)
            // stay with the general function.
            slow |= low & ((m.SLASH << 1) | pM);
            slow |= m.LU & (pLB | pM | (m.SLASH << 1));
            uint64_t und_after = (low | m.LU) & pAPOS & own;                                   // letter right after an apostrophe
            uint64_t und_near = ((low & pL & aposNear) | (m.LU & (pLL | pLU) & aposNear)) & own;  // letter 2-3 bytes after, behind a letter
            uint64_t und_apos = m.APOS & own;
            for (uint64_t aps = m.APOS & (und_apos | (und_after >> 1) | (und_near >> 2) | (und_near >> 3)); aps;) {
                const int j = B2_CTZLL(aps); aps &= aps - 1;
                const uint64_t aj = 1ull << j, p1 = aj >> 1, a1 = aj << 1, a2 = aj << 2, a3 = aj << 3;
                const bool at_d = (m.D & aj) != 0;
                if (!at_d && ((m.M | unk0 | m.SLASH) & p1)) continue;
                bool ba;                                   // does a piece start at the apostrophe
                bool b1 = false, set1 = false, b2 = false, set2 = false, b3 = false, set3 = false;
                if (!at_d && (L & p1)) {
                    if (aposNear & aj) continue;                                                    // a chain
                    if ((m.D & a1) || !(m.valid & a1)) ba = true;                                   // last scalar of its document
                    else {
                        if (m.hi & a1) continue;
                        const bool l1 = (L & a1) != 0;
                        const unsigned c1 = t.text[win0 + j + 1] | 0x20u;
                        const bool sdmt = l1 && (c1 == 's' || c1 == 'd' || c1 == 'm' || c1 == 't');
                        bool two = false;
                        if (l1 && !sdmt && (L & a2) && !(m.hi & a2) && !(m.D & a2)) {
                            const unsigned c2 = t.text[win0 + j + 2] | 0x20u;
                            two = (c1 == 'l' && c2 == 'l') || (c1 == 'v' && c2 == 'e') || (c1 == 'r' && c2 == 'e');
                        }
                        if (sdmt) { ba = false; set1 = true; b1 = false; if ((L & a2) && !(m.D & a2)) { set2 = true; b2 = true; } }
                        else if (two) { ba = false; set1 = true; b1 = false; set2 = true; b2 = false;
                                        if ((L & a3) && !(m.D & a3)) { set3 = true; b3 = true; } }
                        else { ba = true; if (l1) { set1 = true; b1 = false; } }
                    }
                } else {
                    if (at_d || ((m.N | m.WS | m.NL) & p1)) ba = true;
                    else if ((m.SP | m.O | m.APOS) & p1) ba = false;
                    else continue;
                    if ((L & a1) && !(m.D & a1)) { set1 = true; b1 = !ba; }
                }
                if (und_apos & aj) { b = ba ? (b | aj) : (b & ~aj); und_apos &= ~aj; }
                if (und_after & a1) { if (set1) { b = b1 ? (b | a1) : (b & ~a1); und_after &= ~a1; } }
                if (und_near & a2) { if (set2) b = b2 ? (b | a2) : (b & ~a2); und_near &= ~a2; }     // else: an ordinary letter
                if (und_near & a3) { if (set3) b = b3 ? (b | a3) : (b & ~a3); und_near &= ~a3; }
            }
            slow |= und_apos | und_after | und_near;
        }
        slow |= m.M | m.SLASH;
        b |= m.O & (pL | pN | ((m.WS | m.NL) << 1));
        slow |= m.O & (pM | (m.SLASH << 1));
        b |= m.N & ~pN;
        {   // `\p{N}{1,3}`: a digit starts a piece iff the count of digits before it in its run is a
            // multiple of 3.  Runs of ASCII digits that start within the 8-byte look-back are counted with
            // shifts; longer or non-ASCII runs go the slow way.
            const uint64_t A = m.NA;
            // an ASCII digit that starts its run.  A byte whose class is unknown here (continuation bytes of a
            // scalar that begins before the window) may belong to a non-ASCII digit: no known run start after it
            const uint64_t rs = A & ~((m.N | unk0) << 1);
            const uint64_t c1 = A << 1, c2 = c1 & (A << 2), c3 = c2 & (A << 3), c4 = c3 & (A << 4);
            const uint64_t c5 = c4 & (A << 5), c6 = c5 & (A << 6), c7 = c6 & (A << 7);
            const uint64_t k1 = rs << 1, k2 = c1 & (rs << 2), k3 = c2 & (rs << 3), k4 = c3 & (rs << 4);
            const uint64_t k5 = c4 & (rs << 5), k6 = c5 & (rs << 6), k7 = c6 & (rs << 7);
            const uint64_t known = (k1 | k2 | k3 | k4 | k5 | k6 | k7) & ~(m.D | (m.D << 1) | (m.D << 2) | (m.D << 3) |
                                   (m.D << 4) | (m.D << 5) | (m.D << 6));
            (void)c7;
            b |= A & pN & known & (k3 | k6);
            slow |= m.N & pN & ~(A & known);
        }
        b |= m.NL & (pL | pN);
        slow |= m.NL & pM;
        b |= WSnn & ~pWSany;
        b |= WSnn & pWSnn & nextNonWs;
        slow |= WSnn & (pNL | (m.hi & pWSany));
    }
    // anything that touches an undecoded (truncated / unknown) non-ASCII byte goes the slow way
    const uint64_t unk = unk0;
    slow |= unk | (unk << 1) | (unk << 2) | (unk << 3) | (unk >> 1);
    slow &= own;
    b = (b & own & ~slow) | (m.D & OWN);
    if (stats) { stats->positions += (unsigned long long)B2_POPCLL(own); stats->slow += (unsigned long long)B2_POPCLL(slow); }
    slow_out = slow;
    return b;
}

// window bits -> the span's word of the piece-start bitmask (+ the end-of-text sentinel)
B2_HD uint32_t span_word(const TextAccess &t, int64_t w, uint64_t b) {
    const int64_t base = w * 32;
    if (base > t.n) return 0;
    uint32_t word = (uint32_t)(b >> 8);
    if (t.n >= base && t.n < base + 32) word |= 1u << (t.n - base);      // end sentinel
    return word;
}

// one span, start to finish, by one thread (host checks, and the reference for the kernel's warp-cooperative form)
template <int PAT, bool CUT = false>
B2_HD uint32_t span_boundaries(const TextAccess &t, int64_t w, SpanStats *stats = nullptr) {
    uint64_t slow;
    uint64_t b = span_fast<PAT, CUT>(t, w, slow, stats);
    const int64_t win0 = w * 32 - 8;
    for (uint64_t s = slow; s;) {
        const int j = B2_CTZLL(s); s &= s - 1;
        if (boundary_before<PAT>(t, win0 + j)) b |= 1ull << j;
    }
    return span_word(t, w, b);
}

}  // namespace b2bpe
