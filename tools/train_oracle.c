/*
 * train_oracle.c -- CPU restatement of tiktoken's `bpe_train` (tiktoken/_educational.py), TEST INFRASTRUCTURE ONLY.
 *
 * Input: the regex pieces of the corpus in corpus order (the caller splits every document with the C oracle,
 * oracle/bpe_oracle.c).  Output: the merges, each as (left id, right id, id of the merged bytes).  Ids 0..255 are the
 * single bytes; a merge whose bytes are new gets the next id, a merge whose bytes already have an id reuses it (the
 * reference overwrites that key of its dict).  The rules:
 *   - every adjacent pair of every word counts once per occurrence, overlapping pairs included;
 *   - the winner has the highest count; ties go to the pair whose first occurrence comes first (word, then position):
 *     the reference's Counter iterates in insertion order and max() keeps the first maximum;
 *   - the merge applies left to right without overlap in every word.
 * Identical pieces have identical states, so the words are the distinct pieces in order of first appearance, each
 * weighted by its count.  Independent of the GPU trainer: full recount of every word that contains the winner, pair
 * table scan for the maximum, word scan for the first occurrence.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static uint64_t fnv(const uint8_t *p, uint64_t n) {
    uint64_t h = 1469598103934665603ull;
    for (uint64_t i = 0; i < n; i++) { h ^= p[i]; h *= 1099511628211ull; }
    return h ^ (n * 0x9E3779B97F4A7C15ull);
}

/* ---- byte strings -> id, insertion order kept by the id --------------------------------------------------------- */
typedef struct {
    uint8_t *blob; uint64_t blob_n, blob_cap;
    uint64_t *off; uint64_t *len; uint64_t n, cap;          /* string i = blob[off[i] .. off[i] + len[i]) */
    int64_t *slot; uint64_t mask;                           /* hash slots -> string index, -1 empty */
} StrSet;

static int ss_init(StrSet *s, uint64_t want) {
    memset(s, 0, sizeof(*s));
    uint64_t cap = 1024;
    while (cap < want * 2) cap <<= 1;
    s->slot = malloc(cap * sizeof(int64_t)); s->mask = cap - 1;
    s->cap = 1024; s->off = malloc(s->cap * 8); s->len = malloc(s->cap * 8);
    s->blob_cap = 4096; s->blob = malloc(s->blob_cap);
    if (!s->slot || !s->off || !s->len || !s->blob) return -1;
    memset(s->slot, 0xFF, cap * sizeof(int64_t));
    return 0;
}
static void ss_free(StrSet *s) { free(s->blob); free(s->off); free(s->len); free(s->slot); }

static int ss_grow(StrSet *s) {
    uint64_t cap = (s->mask + 1) * 2;
    int64_t *ns = malloc(cap * sizeof(int64_t));
    if (!ns) return -1;
    memset(ns, 0xFF, cap * sizeof(int64_t));
    for (uint64_t i = 0; i < s->n; i++) {
        uint64_t h = fnv(s->blob + s->off[i], s->len[i]) & (cap - 1);
        while (ns[h] >= 0) h = (h + 1) & (cap - 1);
        ns[h] = (int64_t)i;
    }
    free(s->slot); s->slot = ns; s->mask = cap - 1;
    return 0;
}

/* index of p[0..n) (inserted if new: *is_new = 1), -1 out of memory.  `extra` = a second part appended to p. */
static int64_t ss_get(StrSet *s, const uint8_t *p, uint64_t n, const uint8_t *q, uint64_t m, int *is_new) {
    uint8_t *tmp = NULL; const uint8_t *key = p;
    if (m) {
        tmp = malloc(n + m ? n + m : 1);
        if (!tmp) return -1;
        memcpy(tmp, p, n); memcpy(tmp + n, q, m); key = tmp; n += m;
    }
    uint64_t h = fnv(key, n) & s->mask;
    while (s->slot[h] >= 0) {
        const int64_t i = s->slot[h];
        if (s->len[i] == n && memcmp(s->blob + s->off[i], key, n) == 0) { free(tmp); *is_new = 0; return i; }
        h = (h + 1) & s->mask;
    }
    if (s->n == s->cap) {
        s->cap *= 2;
        uint64_t *o = realloc(s->off, s->cap * 8), *l = realloc(s->len, s->cap * 8);
        if (o) s->off = o;
        if (l) s->len = l;
        if (!o || !l) { free(tmp); return -1; }
    }
    while (s->blob_n + n > s->blob_cap) {
        s->blob_cap *= 2;
        uint8_t *b = realloc(s->blob, s->blob_cap);
        if (!b) { free(tmp); return -1; }
        s->blob = b;
    }
    memcpy(s->blob + s->blob_n, key, n);
    s->off[s->n] = s->blob_n; s->len[s->n] = n; s->blob_n += n;
    s->slot[h] = (int64_t)s->n;
    const int64_t id = (int64_t)s->n++;
    free(tmp);
    *is_new = 1;
    if (s->n * 2 > s->mask + 1 && ss_grow(s)) return -1;
    return id;
}

/* ---- (left, right) -> weighted count ------------------------------------------------------------------------------ */
typedef struct { uint64_t *key; int64_t *cnt; uint64_t mask, n; } PairMap;
static const uint64_t EMPTY = ~0ull;

static uint64_t mix(uint64_t k) { k ^= k >> 33; k *= 0xFF51AFD7ED558CCDull; k ^= k >> 33; return k; }

static int pm_init(PairMap *m, uint64_t want) {
    uint64_t cap = 1024;
    while (cap < want * 2) cap <<= 1;
    m->key = malloc(cap * 8); m->cnt = calloc(cap, 8); m->mask = cap - 1; m->n = 0;
    if (!m->key || !m->cnt) return -1;
    memset(m->key, 0xFF, cap * 8);
    return 0;
}
static int pm_add(PairMap *m, uint64_t k, int64_t d) {
    uint64_t h = mix(k) & m->mask;
    while (m->key[h] != EMPTY && m->key[h] != k) h = (h + 1) & m->mask;
    if (m->key[h] == EMPTY) {
        m->key[h] = k; m->n++;
        if (m->n * 2 > m->mask + 1) {           /* rehash at half load */
            const uint64_t cap = (m->mask + 1) * 2;
            uint64_t *nk = malloc(cap * 8); int64_t *nc = calloc(cap, 8);
            if (!nk || !nc) { free(nk); free(nc); return -1; }
            memset(nk, 0xFF, cap * 8);
            m->cnt[h] += d; d = 0;
            for (uint64_t i = 0; i <= m->mask; i++) if (m->key[i] != EMPTY) {
                uint64_t j = mix(m->key[i]) & (cap - 1);
                while (nk[j] != EMPTY) j = (j + 1) & (cap - 1);
                nk[j] = m->key[i]; nc[j] = m->cnt[i];
            }
            free(m->key); free(m->cnt); m->key = nk; m->cnt = nc; m->mask = cap - 1;
            return 0;
        }
    }
    m->cnt[h] += d;
    return 0;
}
static int64_t pm_get(const PairMap *m, uint64_t k) {
    uint64_t h = mix(k) & m->mask;
    while (m->key[h] != EMPTY) { if (m->key[h] == k) return m->cnt[h]; h = (h + 1) & m->mask; }
    return 0;
}

static uint64_t pk(uint32_t a, uint32_t b) { return (uint64_t)a << 32 | b; }

static int word_pairs(PairMap *m, const uint32_t *s, uint32_t n, int64_t d) {
    for (uint32_t i = 0; i + 1 < n; i++) if (pm_add(m, pk(s[i], s[i + 1]), d)) return -1;
    return 0;
}

/* Returns the number of merges (>= 0), -1 when no pair is left before vocab_size is reached, -2 out of memory, -3 more
 * than `cap` merges would be needed.  merges: 3 uint32 per merge.  *n_distinct: distinct words. */
int64_t tro_train(const uint8_t *blob, const uint64_t *piece_off, uint64_t n_pieces, uint32_t vocab_size,
                  uint32_t *merges, uint64_t cap, uint64_t *n_distinct) {
    int64_t rc = -2;
    StrSet words, toks;
    PairMap pm = {0};
    uint64_t *wcnt = NULL, *woff = NULL; uint32_t *wlen = NULL, *sym = NULL;
    int a = ss_init(&words, n_pieces / 4 + 16), b = ss_init(&toks, 4096);
    if (a || b) goto out;
    uint64_t wcap = 1024;
    wcnt = calloc(wcap, 8);
    if (!wcnt) goto out;
    for (uint64_t i = 0; i < n_pieces; i++) {
        int is_new;
        const int64_t w = ss_get(&words, blob + piece_off[i], piece_off[i + 1] - piece_off[i], NULL, 0, &is_new);
        if (w < 0) goto out;
        if ((uint64_t)w >= wcap) {
            uint64_t *t = realloc(wcnt, wcap * 2 * 8);
            if (!t) goto out;
            memset(t + wcap, 0, wcap * 8); wcnt = t; wcap *= 2;
        }
        wcnt[w]++;
    }
    const uint64_t D = words.n;
    *n_distinct = D;
    woff = malloc((D + 1) * 8); wlen = malloc((D + 1) * 4); sym = malloc((words.blob_n + 1) * 4);
    if (!woff || !wlen || !sym) goto out;
    uint64_t P0 = 0;
    for (uint64_t w = 0; w < D; w++) {
        woff[w] = words.off[w]; wlen[w] = (uint32_t)words.len[w];
        for (uint64_t j = 0; j < words.len[w]; j++) sym[woff[w] + j] = words.blob[words.off[w] + j];
        P0 += words.len[w];
    }
    if (pm_init(&pm, P0 + 16)) goto out;
    for (uint64_t w = 0; w < D; w++) if (word_pairs(&pm, sym + woff[w], wlen[w], (int64_t)wcnt[w])) goto out;
    for (int i = 0; i < 256; i++) { uint8_t c = (uint8_t)i; int is_new; if (ss_get(&toks, &c, 1, NULL, 0, &is_new) != i) goto out; }
    uint64_t nm = 0;
    while (toks.n < vocab_size) {
        int64_t best = 0;
        for (uint64_t i = 0; i <= pm.mask; i++) if (pm.key[i] != EMPTY && pm.cnt[i] > best) best = pm.cnt[i];
        if (best == 0) { rc = -1; goto out; }
        uint32_t L = 0, R = 0; int found = 0;
        for (uint64_t w = 0; w < D && !found; w++)
            for (uint32_t i = 0; i + 1 < wlen[w]; i++) {
                const uint32_t *s = sym + woff[w];
                if (pm_get(&pm, pk(s[i], s[i + 1])) == best) { L = s[i]; R = s[i + 1]; found = 1; break; }
            }
        if (!found) { rc = -2; goto out; }
        if (nm == cap) { rc = -3; goto out; }
        int is_new;
        const int64_t id = ss_get(&toks, toks.blob + toks.off[L], toks.len[L], toks.blob + toks.off[R], toks.len[R], &is_new);
        if (id < 0) goto out;
        merges[3 * nm] = L; merges[3 * nm + 1] = R; merges[3 * nm + 2] = (uint32_t)id; nm++;
        for (uint64_t w = 0; w < D; w++) {
            uint32_t *s = sym + woff[w]; const uint32_t n = wlen[w];
            uint32_t i = 0;
            while (i + 1 < n && !(s[i] == L && s[i + 1] == R)) i++;
            if (i + 1 >= n) continue;
            if (word_pairs(&pm, s, n, -(int64_t)wcnt[w])) goto out;
            uint32_t o = 0;
            for (i = 0; i < n;) {
                if (i + 1 < n && s[i] == L && s[i + 1] == R) { s[o++] = (uint32_t)id; i += 2; }
                else s[o++] = s[i++];
            }
            wlen[w] = o;
            if (word_pairs(&pm, s, o, (int64_t)wcnt[w])) goto out;
        }
    }
    rc = (int64_t)nm;
out:
    ss_free(&words); ss_free(&toks);
    free(pm.key); free(pm.cnt); free(wcnt); free(woff); free(wlen); free(sym);
    return rc;
}
