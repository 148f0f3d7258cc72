// bpe_tables.h -- host-side construction of the engine's lookup tables from mergeable_ranks.
// Replaces CoreBPE::new_internal's map building (src/lib.rs:618-663): runs once per Encoding.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "bpe_device.cuh"

namespace b2bpe {

struct HostTables {
    std::vector<uint32_t> byte_id;    // 256
    std::vector<uint32_t> pair2;      // 65536
    std::vector<U4> pair_tab;   uint32_t pair_mask = 0;
    std::vector<U4> narrow_tab; uint32_t narrow_mask = 0;
    std::vector<U4> wide_tab;   uint32_t wide_mask = 0;
    std::vector<U4> long_tab;   uint32_t long_mask = 0;
    std::vector<uint8_t> long_blob;
    uint32_t max_token_len = 0, n_long_tokens = 0, max_rank = 0;
    uint64_t n_pairs = 0;
    // decode side (host): rank -> bytes
    std::unordered_map<uint32_t, std::string> decoder;
    std::string error;

    DevTables view() const {
        DevTables T;
        T.byte_id = byte_id.data(); T.pair2 = pair2.data();
        T.pair_tab = pair_tab.data(); T.pair_mask = pair_mask;
        T.narrow_tab = narrow_tab.data(); T.narrow_mask = narrow_mask;
        T.wide_tab = wide_tab.data(); T.wide_mask = wide_mask;
        T.long_tab = long_tab.data(); T.long_mask = long_mask;
        T.long_blob = long_blob.data();
        T.max_token_len = max_token_len; T.n_long_tokens = n_long_tokens;
        return T;
    }
};

inline uint32_t pow2_at_least(uint64_t n) { uint32_t c = 16; while (c < n) c <<= 1; return c; }

inline void pack16(const uint8_t *p, uint32_t len, uint64_t &k0, uint64_t &k1) {
    uint8_t b[16] = {0};
    memcpy(b, p, len);
    memcpy(&k0, b, 8); memcpy(&k1, b + 8, 8);       // little-endian hosts only (x86-64, aarch64)
}

inline uint64_t long_hash_bytes(const uint8_t *p, uint32_t len) {
    uint64_t h = long_hash_init(len);
    for (uint32_t i = 0; i < len; i += 8) {
        uint8_t b[8] = {0};
        memcpy(b, p + i, len - i < 8 ? len - i : 8);
        uint64_t w; memcpy(&w, b, 8);
        h = long_hash_step(h, w, i / 8);
    }
    return h;
}

// returns 0 or a negative B200BPE_E* code (values mirrored from include/b200bpe.h)
inline int build_tables(const uint8_t *tok_bytes, const uint64_t *tok_off, const uint32_t *tok_rank,
                        uint32_t n, HostTables &H) {
    std::unordered_map<std::string, uint32_t> enc;
    enc.reserve((size_t)n * 2 + 16);
    H.decoder.reserve((size_t)n * 2 + 16);
    for (uint32_t i = 0; i < n; i++) {
        uint64_t len = tok_off[i + 1] - tok_off[i];
        if (len == 0) { H.error = "empty token in mergeable_ranks"; return -1; }
        if (tok_rank[i] >= (1u << 30)) { H.error = "rank too large (token ids must be < 2^30)"; return -1; }
        std::string s((const char *)tok_bytes + tok_off[i], (size_t)len);
        if (!enc.emplace(s, tok_rank[i]).second) { H.error = "duplicate token bytes"; return -1; }
        if (!H.decoder.emplace(tok_rank[i], s).second) {
            // reference: assert!(encoder.len() == decoder.len(), ...) src/lib.rs:636-641
            H.error = "Encoder and decoder must be of equal length. Maybe you had duplicate token indices in your encoder?";
            return -3;
        }
        if (len > H.max_token_len) H.max_token_len = (uint32_t)len;
        if (tok_rank[i] > H.max_rank) H.max_rank = tok_rank[i];
    }
    H.byte_id.assign(256, 0);
    for (int b = 0; b < 256; b++) {
        auto it = enc.find(std::string(1, (char)b));
        H.byte_id[b] = it != enc.end() ? it->second : PSEUDO_BASE + (uint32_t)b;
    }
    H.pair2.assign(65536, RANK_MAX);
    auto id_of = [&](const std::string &s, uint32_t &id) -> bool {
        auto it = enc.find(s);
        if (it != enc.end()) { id = it->second; return true; }
        if (s.size() == 1) { id = PSEUDO_BASE + (uint8_t)s[0]; return true; }
        return false;
    };
    struct Pair { uint32_t a, b, r; };
    std::vector<Pair> pairs;
    uint32_t n_narrow = 0, n_wide = 0, n_long = 0;
    for (auto &kv : enc) {
        const std::string &t = kv.first;
        if (t.size() <= (size_t)NARROW_MAX) n_narrow++; else if (t.size() <= (size_t)SHORT_MAX) n_wide++; else n_long++;
        if (t.size() == 2) H.pair2[((uint8_t)t[0] << 8) | (uint8_t)t[1]] = kv.second;
        for (size_t k = 1; k < t.size(); k++) {
            uint32_t a, b;
            if (id_of(t.substr(0, k), a) && id_of(t.substr(k), b)) pairs.push_back({a, b, kv.second});
        }
    }
    H.n_pairs = pairs.size();
    // Keys go in in ascending rank order (ties by key, so the layout is deterministic): under linear probing the first
    // key to reach a slot keeps it, so the low ranks -- the frequent tokens and merges of a BPE vocabulary -- sit in
    // their home slot and are found with one load.
    std::sort(pairs.begin(), pairs.end(), [](const Pair &x, const Pair &y) {
        return x.r != y.r ? x.r < y.r : x.a != y.a ? x.a < y.a : x.b < y.b;
    });
    // linear probing over single slots; capacity >= 3 x the entries (load <= 1/3).  Word w of a slot
    // is 1 when the probe path of some key passes through it (the key lives further on): a slot without that mark that
    // does not hold the key ends the chain, so an absent pair usually costs one load even when its home slot is taken.
    uint32_t nslots = pow2_at_least((uint64_t)pairs.size() * 3 + 2);
    H.pair_mask = nslots - 1;
    H.pair_tab.assign((size_t)nslots, U4{PAIR_EMPTY, PAIR_EMPTY, RANK_MAX, 0});
    for (auto &p : pairs) {
        uint32_t s = pair_hash(p.a, p.b) & H.pair_mask;
        while (H.pair_tab[s].x != PAIR_EMPTY) { H.pair_tab[s].w = 1; s = (s + 1) & H.pair_mask; }
        H.pair_tab[s] = U4{p.a, p.b, p.r, 0};
    }
    // piece tables, load <= 1/3 each: narrow (1..11 bytes) one U4 per slot, wide (12..16 bytes) two
    uint32_t nc = pow2_at_least((uint64_t)n_narrow * 3 + 2);
    H.narrow_mask = nc - 1;
    H.narrow_tab.assign((size_t)nc, U4{0, 0, 0, 0});
    uint32_t wc = pow2_at_least((uint64_t)n_wide * 3 + 2);
    H.wide_mask = wc - 1;
    H.wide_tab.assign((size_t)wc * 2, U4{0, 0, 0, 0});
    uint32_t lc = pow2_at_least((uint64_t)n_long * 2 + 2);
    H.long_mask = lc - 1;
    H.long_tab.assign((size_t)lc * 2, U4{0, 0, 0, 0});
    H.n_long_tokens = n_long;
    std::vector<std::pair<uint32_t, const std::string *>> by_rank;   // ascending rank, as for the pairs
    by_rank.reserve(enc.size());
    for (auto &kv : enc) by_rank.emplace_back(kv.second, &kv.first);
    std::sort(by_rank.begin(), by_rank.end());
    for (auto &rt : by_rank) {
        const std::string &t = *rt.second;
        const uint32_t rank = rt.first;
        uint32_t len = (uint32_t)t.size();
        if (len <= NARROW_MAX) {                   // byte 11 of the key is zero padding: it carries the length
            uint64_t k0, k1; pack16((const uint8_t *)t.data(), len, k0, k1);
            uint32_t s = piece_hash(k0, k1, len) & H.narrow_mask;
            while (H.narrow_tab[s].z != 0) { H.narrow_tab[s].w |= PIECE_THROUGH; s = (s + 1) & H.narrow_mask; }
            H.narrow_tab[s] = U4{(uint32_t)k0, (uint32_t)(k0 >> 32), (uint32_t)k1 | len << 24, rank};
        } else if (len <= (uint32_t)SHORT_MAX) {          // both piece tables carry the pass-through mark of the pair table
            uint64_t k0, k1; pack16((const uint8_t *)t.data(), len, k0, k1);
            uint32_t s = piece_hash(k0, k1, len) & H.wide_mask;
            while (H.wide_tab[2 * s + 1].x != 0) { H.wide_tab[2 * s + 1].z = 1; s = (s + 1) & H.wide_mask; }
            H.wide_tab[2 * s] = U4{(uint32_t)k0, (uint32_t)(k0 >> 32), (uint32_t)k1, (uint32_t)(k1 >> 32)};
            H.wide_tab[2 * s + 1] = U4{len, rank, 0, 0};
        } else {
            uint64_t h = long_hash_bytes((const uint8_t *)t.data(), len);
            uint32_t s = (uint32_t)(h ^ (h >> 32)) & H.long_mask;
            while (H.long_tab[2 * s].w != 0) s = (s + 1) & H.long_mask;
            uint32_t off = (uint32_t)H.long_blob.size();
            H.long_blob.insert(H.long_blob.end(), t.begin(), t.end());
            H.long_tab[2 * s] = U4{(uint32_t)h, (uint32_t)(h >> 32), off, len};
            H.long_tab[2 * s + 1] = U4{rank, 0, 0, 0};
        }
    }
    if (H.long_blob.empty()) H.long_blob.push_back(0);
    return 0;
}

}  // namespace b2bpe
