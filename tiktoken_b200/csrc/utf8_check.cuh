// utf8_check.cuh -- UTF-8 well-formedness of packed documents, one 32-byte span at a time (bytes mode,
// b200bpe_encode_bytes_batch).  Host + device: hostcheck.cpp runs the same function on the CPU.
//
// The well-formed sequences are those of Unicode Table 3-7, which std::str::from_utf8 (src/py.rs:74) accepts:
//   C2..DF 80..BF | E0 A0..BF 80..BF | E1..EC,EE..EF 80..BF 80..BF | ED 80..9F 80..BF
//   F0 90..BF 80..BF 80..BF | F1..F3 80..BF 80..BF 80..BF | F4 80..8F 80..BF 80..BF
// A sequence never crosses a document start.  A position is marked when it is the first byte of an ill-formed
// sequence: a lead whose sequence is not well-formed, a continuation byte that no well-formed sequence covers, or
// one of C0, C1, F5..FF.  Decoding left to right, everything before the first mark of a document is well-formed and
// the decoder fails at that mark, so the first mark is `valid_up_to`.
#pragma once
#include "text_access.cuh"

namespace b2bpe {

// bit j: byte w * 32 + j starts an ill-formed sequence.  Reads bytes [w*32 - 8, w*32 + 56) of text (bytes at or past n
// count as absent) and doc-start words w - 1 .. w + 1.
B2_HD uint32_t utf8_bad_word(const uint8_t *text, int64_t n, const uint32_t *dbits, int64_t w) {
    const int64_t win0 = w * 32 - 8;                      // window bit j = byte win0 + j; own bytes are bits 8..39
    uint32_t W[16];
#if defined(__CUDA_ARCH__)
    if (win0 >= 0 && win0 + 64 <= n) {
        const uint2 *p = reinterpret_cast<const uint2 *>(text + win0);
#pragma unroll
        for (int k = 0; k < 8; k++) { const uint2 v = __ldg(p + k); W[2 * k] = v.x; W[2 * k + 1] = v.y; }
    } else
#endif
    {
        for (int k = 0; k < 16; k++) {
            uint32_t x = 0;
            for (int b = 0; b < 4; b++) {
                const int64_t pos = win0 + 4 * k + b;
                if (pos >= 0 && pos < n) x |= (uint32_t)text[pos] << (8 * b);
            }
            W[k] = x;
        }
    }
    uint32_t any = 0;
    for (int k = 0; k < 16; k++) any |= W[k];
    if (!(any & 0x80808080u)) return 0;                  // all ASCII: nothing can be ill-formed
    uint64_t V = 0, C = 0, L2 = 0, L3 = 0, L4 = 0, BAD = 0, E0 = 0, ED = 0, F0 = 0, F4 = 0;
    uint64_t CA = 0, CB = 0, CC = 0, CD = 0;             // continuation bytes A0..BF, 80..9F, 90..BF, 80..8F
    for (int j = 0; j < 64; j++) {
        const int64_t pos = win0 + j;
        if (pos < 0 || pos >= n) continue;
        const uint64_t bit = 1ull << j;
        const uint32_t b = (W[j >> 2] >> (8 * (j & 3))) & 0xFFu;
        V |= bit;
        if (b < 0x80u) continue;
        if (b < 0xC0u) {
            C |= bit;
            if (b >= 0xA0u) CA |= bit; else CB |= bit;
            if (b >= 0x90u) CC |= bit; else CD |= bit;
        } else if (b < 0xC2u) BAD |= bit;
        else if (b < 0xE0u) L2 |= bit;
        else if (b < 0xF0u) { L3 |= bit; if (b == 0xE0u) E0 |= bit; if (b == 0xEDu) ED |= bit; }
        else if (b < 0xF5u) { L4 |= bit; if (b == 0xF0u) F0 |= bit; if (b == 0xF4u) F4 |= bit; }
        else BAD |= bit;
    }
    uint64_t D = (uint64_t)dbits[w] << 8;                 // document starts of the window
    if (w > 0) D |= (uint64_t)(dbits[w - 1] >> 24);
    D |= (uint64_t)dbits[w + 1] << 40;
    const uint64_t Cin = C & V & ~D;                      // a continuation byte of the same document as the byte before
    const uint64_t S2 = (Cin >> 1) & ~(E0 & ~(CA >> 1)) & ~(ED & ~(CB >> 1)) & ~(F0 & ~(CC >> 1)) & ~(F4 & ~(CD >> 1));
    const uint64_t VS2 = L2 & S2, VS3 = L3 & S2 & (Cin >> 2), VS4 = L4 & S2 & (Cin >> 2) & (Cin >> 3);
    const uint64_t VS = VS2 | VS3 | VS4;                  // well-formed sequence starts
    const uint64_t covered = (VS << 1) | ((VS3 | VS4) << 2) | (VS4 << 3);
    const uint64_t bad = ((C & ~covered) | ((L2 | L3 | L4) & ~VS) | BAD) & V;
    return (uint32_t)(bad >> 8);
}

}  // namespace b2bpe
