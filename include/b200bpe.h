/*
 * b200bpe.h -- C ABI of libb200bpe.so, the H100-native BPE encoder that replaces tiktoken's
 * Rust extension `_tiktoken` (reference: openai/tiktoken v0.14.0, src/lib.rs + src/py.rs).
 *
 * Boundary: this is exactly what a `_tiktoken` replacement binds.  Each entry point names the
 * reference interface it stands in for (file:line in /root/reference).  Plain pointers and
 * sizes only; no torch / Python types.  All functions return 0 on success and a negative
 * B200BPE_E* code on failure; `b200bpe_last_error()` returns a thread-local message.
 *
 * There is no CPU fallback: every encode call runs the sm_90a kernels on the device the
 * engine was created on, and fails with B200BPE_ECUDA if that is not possible.
 */
#ifndef B200BPE_H
#define B200BPE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200BPE_OK        0
#define B200BPE_EINVAL   -1   /* bad argument (-> ValueError)                                  */
#define B200BPE_EPATTERN -2   /* pat_str is not one of the three supported patterns (ValueError;
                                 the reference raises ValueError for an invalid regex, py.rs:21-22) */
#define B200BPE_EDUPRANK -3   /* duplicate rank in mergeable_ranks (reference: assert, lib.rs:636-641) */
#define B200BPE_ECUDA    -4   /* CUDA error / no device (-> RuntimeError)                      */
#define B200BPE_ENOBYTE  -5   /* a piece needed a single-byte token the vocabulary lacks
                                 (reference: `ranks[...]` index panic, lib.rs:202,207)         */
#define B200BPE_EKEY     -6   /* unknown token id in decode (-> KeyError, py.rs:160)           */
#define B200BPE_ESPECIAL -7   /* the text contains a disallowed special token (-> ValueError,
                                 tiktoken/core.py:120-124, :431-438)                           */
#define B200BPE_ECAPACITY -8  /* a device work-space had to grow while several asynchronous device
                                 calls were queued: re-issue them (b200bpe_device_wait); training: more
                                 merges than the caller's merge buffer holds                      */
#define B200BPE_ENOPAIR  -9   /* training: no pair is left to merge before vocab_size is reached (-> ValueError;
                                 the reference's max() of an empty Counter, tiktoken/_educational.py:144) */

typedef struct b200bpe b200bpe_t;
typedef struct b200bpe_result b200bpe_result_t;

/* CoreBPE::new / py_new (src/lib.rs:601-663, src/py.rs:15-23).
 * mergeable_ranks is passed flattened: token i has bytes tok_bytes[tok_off[i] .. tok_off[i+1]) and
 * rank tok_rank[i]; special tokens likewise (UTF-8 strings).  pat_str must be one of the three
 * pat_strs of tiktoken_ext/openai_public.py (:12-14, :89, :104-114).  Builds the device tables
 * (rank tables, pair table, Unicode class tables) on CUDA device `device`. */
int b200bpe_create(const uint8_t *tok_bytes, const uint64_t *tok_off, const uint32_t *tok_rank,
                   uint32_t n_tok,
                   const uint8_t *sp_bytes, const uint64_t *sp_off, const uint32_t *sp_rank,
                   uint32_t n_sp,
                   const char *pat_str, int device, b200bpe_t **out);

/* The same constructor for ONE engine spread over several GPUs of the box (SURVEY.md 8(b): `const int* devices,
 * int n_dev`): the tables are replicated on every listed device; the host-buffer entry points below cut a batch into
 * chunks that go round-robin over the devices and place every chunk's tokens at its final offset of one pinned result
 * buffer -- the count "gather" is a host prefix sum, no token payload crosses NVLink.  Chunks end at document boundaries
 * (documents are independent haystacks, src/lib.rs:360-373) and, in the encode and count entry points, also at seams
 * inside documents larger than two chunks: a space between two ASCII letters, or a '\n' between a printable ASCII
 * character and an ASCII letter or digit, where the split into pieces is provably that of the whole document, so
 * outputs are unchanged (b200bpe_last_doc_seams).  The device-resident entry points use devices[0]. */
int b200bpe_create_multi(const uint8_t *tok_bytes, const uint64_t *tok_off, const uint32_t *tok_rank,
                         uint32_t n_tok,
                         const uint8_t *sp_bytes, const uint64_t *sp_off, const uint32_t *sp_rank,
                         uint32_t n_sp,
                         const char *pat_str, const int *devices, int n_dev, b200bpe_t **out);

/* Number of devices an engine runs on. */
int b200bpe_n_devices(b200bpe_t *h);

/* Release the grow-only device work-spaces (~25 bytes per input byte of the largest batch seen, per pipeline slot)
 * and the pooled pinned result blocks; the tables stay and the next call re-allocates what it needs. */
int b200bpe_trim(b200bpe_t *h);

/* Outstanding results keep the engine alive: with results not yet freed this only marks the handle dead and the
 * last b200bpe_result_free tears it down (TiktokenBuffer owns its Vec in the reference, src/py.rs:186-189). */
void b200bpe_destroy(b200bpe_t *h);

/* The batched form of CoreBPE::encode_ordinary (src/lib.rs:360-373, py.rs:29-32) as fanned out
 * by Encoding.encode_ordinary_batch (tiktoken/core.py:164-176): ONE native call for the whole
 * batch.  text = concatenated UTF-8 of all documents, document d = [doc_off[d], doc_off[d+1]).
 * HOST buffers; the call copies them to the device, runs the kernels and brings back tokens
 * (uint32[n_tokens], documents concatenated) and offsets (uint64[n_docs+1]).  A document may have any length: one
 * larger than two chunks is cut only at seams (see b200bpe_create_multi), which leaves the output unchanged; only a stretch
 * of 4 GiB or more without a seam is refused (B200BPE_EINVAL).  The same holds for b200bpe_encode_batch,
 * b200bpe_encode_batch_special and b200bpe_count_batch, whose seams also never fall inside a flagged special token. */
int b200bpe_encode_ordinary_batch(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off,
                                  uint64_t n_docs, b200bpe_result_t **out);

/* The batched form of CoreBPE::encode (src/lib.rs:375-442, py.rs:34-49) as fanned out by
 * Encoding.encode_batch (core.py:178-206).  allowed[i] != 0 marks special token i (index into
 * the arrays given to b200bpe_create) as allowed; allowed == NULL means none (then identical to
 * the ordinary form).  Allowed specials split each document into separate haystacks
 * (lib.rs:402-405) and are emitted as their own ids (lib.rs:426-436). */
int b200bpe_encode_batch(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs,
                         const uint8_t *allowed, b200bpe_result_t **out);

/* CoreBPE::encode (src/lib.rs:375-442) together with the disallowed-special check that Encoding.encode /
 * encode_batch run first (tiktoken/core.py:120-124, :197-204, :431-438), both as ONE multi-pattern scan on the device.
 * flags[i] for special token i (index into the arrays given to b200bpe_create): 1 = allowed (cuts its document into
 * haystacks, emitted as its own id), 2 = disallowed (its presence anywhere fails the call with B200BPE_ESPECIAL and
 * *special_index = the leftmost offending special), 0 = ordinary text.  flags == NULL: no special handling.  Long
 * documents as in b200bpe_encode_ordinary_batch: cut only at seams outside every flagged special, outputs unchanged. */
int b200bpe_encode_batch_special(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs,
                                 const uint8_t *flags, b200bpe_result_t **out, int32_t *special_index);

/* Token counts of CoreBPE::encode for every document, without the tokens: tok_off[n_docs+1] (HOST, caller-owned)
 * receives exactly the offsets b200bpe_encode_batch_special returns for the same text, doc_off and flags, so document
 * d has tok_off[d+1] - tok_off[d] tokens.  flags as in b200bpe_encode_batch_special (NULL: ordinary); a disallowed
 * special fails with B200BPE_ESPECIAL and *special_index = the leftmost one.  No token leaves the device, and neither
 * the device output token buffer (4 bytes per input byte) nor a pinned token block is allocated; the long-piece and
 * special-token work-space (another 4 bytes per input byte) still is.  Long documents as in
 * b200bpe_encode_batch_special. */
int b200bpe_count_batch(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs,
                        const uint8_t *flags, uint64_t *tok_off, int32_t *special_index);

/* CoreBPE::_encode_bytes (src/py.rs:72-115, Encoding._encode_bytes in tiktoken/core.py) for every document of a batch:
 * the documents need not be UTF-8.  A document that is well-formed UTF-8 gets exactly the tokens of
 * b200bpe_encode_ordinary_batch.  For any other, with v = its std::str::from_utf8 valid_up_to: its first v bytes are
 * encoded as their own haystack (special-token text is ordinary text), the tokens of their last regex piece are dropped
 * (together with the all-space tokens before them when the first of them is all-space, lib.rs:444-481) and the dropped
 * bytes plus everything from v on are encoded as ONE piece (whole-piece probe, then byte_pair_encode).  A missing
 * single-byte token fails with B200BPE_ENOBYTE.  Same buffers and result as b200bpe_encode_ordinary_batch.  Needs every
 * token id below 2^24 (the device decode tables give the token lengths), else B200BPE_EINVAL. */
int b200bpe_encode_bytes_batch(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs,
                               b200bpe_result_t **out);

/* Encoding.encode_with_unstable (tiktoken/core.py:208-243 -> src/py.rs:117-131 -> CoreBPE::_encode_unstable_native,
 * src/lib.rs:483-599) for every document of a batch, with the flags and the disallowed check of
 * b200bpe_encode_batch_special (B200BPE_ESPECIAL, *special_index = the leftmost offender).  Per document: the tokens of
 * CoreBPE::encode (lib.rs:375-442) minus those of the last regex piece of its final haystack (none when the document is
 * empty or ends with an allowed special, lib.rs:430-433), extended backwards over all-space mergeable tokens
 * (lib.rs:444-481) -- the stable tokens, in *stable like b200bpe_encode_batch_special's result --, and the completions of
 * the unstable bytes U they covered: (a) every token that starts with U (lib.rs:537-549); (b) for i = 1 .. |U|-1 and every
 * token t that starts with U[i:], encode_ordinary(U[:i] + t) when that is UTF-8, else byte_pair_encode of it, cut after the
 * first token at which the byte count reaches |U| (lib.rs:551-584); (c) when |U| > 1 and U ends in a White_Space scalar
 * after other bytes, byte_pair_encode(front) + byte_pair_encode(last scalar) (lib.rs:586-596).  Each distinct completion
 * of a document comes once, at its first position in that order (the reference returns a HashSet).
 * *completions: b200bpe_result_tokens = every completion's tokens back to back, b200bpe_result_offsets = their
 * boundaries (b200bpe_result_n_docs() + 1 of them), b200bpe_result_groups = per input document the range of its
 * completions (n_docs + 1).  A missing single-byte token fails with B200BPE_ENOBYTE; every token id must be < 2^24
 * (the device decode tables give the token bytes), else B200BPE_EINVAL.  Candidate text goes through the encoder in
 * rounds of at most one chunk (B200BPE_CHUNK_MB). */
int b200bpe_encode_with_unstable_batch(b200bpe_t *h, const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs,
                                       const uint8_t *flags, b200bpe_result_t **stable, b200bpe_result_t **completions,
                                       int32_t *special_index);

/* tiktoken._educational.bpe_train (tiktoken/_educational.py:119-185) over a batch of documents; needs no engine.
 * text = concatenated UTF-8 of all documents, document d = [doc_off[d], doc_off[d+1]) (HOST buffers).  The words are the
 * pat_str pieces of document 0, then document 1, ... (no piece crosses a document boundary).  pat_str must be one of the
 * three patterns b200bpe_create accepts.  Starting from the 256 single bytes, each merge takes the adjacent pair of
 * highest count over all words (ties: the pair whose first occurrence comes first, by word, then position), applies it
 * left to right without overlap in every word, and gives the merged bytes the id len(ranks) -- or, when those bytes
 * already are a token, that token's id, and len(ranks) does not grow -- until len(ranks) == vocab_size.
 * merges_out receives 3 uint32 per merge: left id, right id, merged id (ids 0..255 are the bytes; a new id is the number
 * of tokens so far); *n_merges_out their count.  At most merges_cap merges, else B200BPE_ECAPACITY.  No pair left
 * before vocab_size: B200BPE_ENOPAIR.  vocab_size < 256: B200BPE_EINVAL.  Runs on CUDA device `device`, the merge loop
 * without a host synchronisation per merge (a CUDA graph of 128 merges per host check).  stats8 (may be NULL): [0] pieces, [1] distinct words, [2] merges, [3] graph batches, device ms of [4] the
 * split, [5] the distinct-word stage, [6] the merge loop, [7] chunks (B200BPE_CHUNK_MB, default 64 MiB). */
int b200bpe_bpe_train(const uint8_t *text, const uint64_t *doc_off, uint64_t n_docs, const char *pat_str,
                      uint32_t vocab_size, int device, uint32_t *merges_out, uint64_t merges_cap,
                      uint64_t *n_merges_out, double *stats8);

/* Name of special token `index` (as given to b200bpe_create), or NULL. */
const char *b200bpe_special_name(b200bpe_t *h, int32_t index);

/* Device-resident form of the same path, for measurement and for callers that already hold the
 * corpus in HBM: d_text (n_bytes, readable up to n_bytes+16), d_doc_off (n_docs+1), outputs
 * d_tokens (capacity n_bytes uint32) and d_tok_off (n_docs+1) are DEVICE pointers on the
 * engine's device; n_tokens is a host pointer.  `stream` is a cudaStream_t (NULL = engine stream).
 * The call returns after the stream has been synchronised. */
int b200bpe_encode_device(b200bpe_t *h, const uint8_t *d_text, uint64_t n_bytes,
                          const uint64_t *d_doc_off, uint64_t n_docs,
                          uint32_t *d_tokens, uint64_t *d_tok_off, uint64_t *n_tokens, void *stream);

/* The same, split in two so that a stream of batches never stops for the host: `_async` only enqueues the kernels on
 * `stream` (no synchronisation; d_counts, if not NULL, is a DEVICE uint64[2] that receives {n_tokens, n_docs} at the
 * end of the pipeline, e.g. as the send buffer of an NCCL all-gather enqueued behind it); `b200bpe_device_wait`
 * waits for the most recent call, returns its token count and reports errors.  Work-spaces are sized from
 * experience, not for the worst case: if one was too small the wait re-runs the LAST call after growing it; with
 * several calls queued that is reported as B200BPE_ECAPACITY (issue a synchronous call first to settle the sizes). */
int b200bpe_encode_device_async(b200bpe_t *h, const uint8_t *d_text, uint64_t n_bytes,
                                const uint64_t *d_doc_off, uint64_t n_docs,
                                uint32_t *d_tokens, uint64_t *d_tok_off, uint64_t *d_counts, void *stream);
int b200bpe_device_wait(b200bpe_t *h, uint64_t *n_tokens);

/* b200bpe_encode_device_async with the special-token policy of b200bpe_encode_batch_special: flags (HOST, one per
 * special token; NULL: ordinary) is copied by the call.  d_tokens == NULL: count only -- d_tok_off and d_counts receive
 * what a call with tokens would give them, no token is written and d_tokens needs no capacity. */
int b200bpe_encode_device_special_async(b200bpe_t *h, const uint8_t *d_text, uint64_t n_bytes,
                                        const uint64_t *d_doc_off, uint64_t n_docs, const uint8_t *flags,
                                        uint32_t *d_tokens, uint64_t *d_tok_off, uint64_t *d_counts, void *stream);
/* b200bpe_device_wait that also reports a disallowed special: B200BPE_ESPECIAL with *special_index (may be NULL) = the
 * leftmost disallowed special of the earliest call of the waited-for series that has one. */
int b200bpe_device_wait_special(b200bpe_t *h, uint64_t *n_tokens, int32_t *special_index);

/* CoreBPE::encode_single_piece (src/py.rs:145-150): BPE of raw bytes without the regex split. */
int b200bpe_encode_single_piece(b200bpe_t *h, const uint8_t *piece, uint64_t len, b200bpe_result_t **out);

/* Result accessors: the buffers stay valid until b200bpe_result_free (the analogue of
 * TiktokenBuffer keeping its Vec<Rank> alive, src/py.rs:186-249). */
const uint32_t *b200bpe_result_tokens(const b200bpe_result_t *r);
const uint64_t *b200bpe_result_offsets(const b200bpe_result_t *r);
uint64_t b200bpe_result_n_tokens(const b200bpe_result_t *r);
/* The completions result of b200bpe_encode_with_unstable_batch: per input document d, its completions are
 * [groups[d], groups[d+1]); *n_groups = the number of input documents.  NULL (and 0) for every other result. */
const uint64_t *b200bpe_result_groups(const b200bpe_result_t *r, uint64_t *n_groups);
uint64_t b200bpe_result_n_docs(const b200bpe_result_t *r);
void b200bpe_result_free(b200bpe_result_t *r);

/* CoreBPE::decode_bytes (src/lib.rs:345-358, py.rs:156-162): gather of token byte strings.
 * Host-side table read (not on the encode hot path).  On an unknown id returns B200BPE_EKEY
 * and stores the id in *bad_token.  out_len receives the byte count; pass out == NULL to size. */
int b200bpe_decode_bytes(b200bpe_t *h, const uint32_t *tokens, uint64_t n_tokens, uint8_t *out,
                         uint64_t out_cap, uint64_t *out_len, uint32_t *bad_token);

/* Batched decode on the device ("next" row): CoreBPE::decode_bytes (src/lib.rs:345-358) as fanned out
 * by Encoding.decode_bytes_batch (tiktoken/core.py:345-350).  HOST buffers: tokens of all documents
 * concatenated, tok_off[n_docs+1].  The result reuses b200bpe_result: b200bpe_result_tokens() points
 * at the BYTES (b200bpe_result_n_tokens() = byte count), b200bpe_result_offsets() at the per-document
 * byte offsets.  Unknown id -> B200BPE_EKEY with *bad_token set (KeyError, py.rs:160). */
int b200bpe_decode_batch(b200bpe_t *h, const uint32_t *tokens, const uint64_t *tok_off, uint64_t n_docs,
                         b200bpe_result_t **out, uint32_t *bad_token);

/* Per-stage device timings (ms, CUDA events on the engine stream) of the most recent encode
 * call on this handle: [0] mark documents, [1] pre-tokenise, [2] long-piece scan + merge,
 * [3] encode stage (probe + miss sort + miss merge), [4] total device time, [5] H2D, [6] D2H,
 * [7] count scan + gather, [8] probe kernel alone.  Also the kernel launch count. */
int b200bpe_last_timings(b200bpe_t *h, float *ms9, uint32_t *n_launches);

/* What the most recent encode call on this handle had to redo: `grown` = OR of B200BPE_GREW_* for the work-spaces this
 * call grew and re-ran, `reruns` = pipeline re-runs summed over chunks and devices, `token_passes` = 1, or 2 when the
 * host token buffer had to be re-sized.  Every encode entry point, b200bpe_encode_device_async and b200bpe_device_wait
 * included, resets all three to 0 first, so a call that fails early reports zeros.  A work-space that was too small for
 * an EARLIER call of a queued device series is not grown (that series fails with B200BPE_ECAPACITY) and is not in
 * `grown`. */
#define B200BPE_GREW_MISS 1u   /* miss queue or miss result space */
#define B200BPE_GREW_SLOW 2u   /* undecided pre-tokeniser positions */
#define B200BPE_GREW_LONG 4u   /* long-piece merge scratch */
int b200bpe_last_reruns(b200bpe_t *h, uint32_t *grown, uint32_t *reruns, uint32_t *token_passes);

/* Which long-piece merge kernels the most recent encode call on this handle ran: counts[c] = pieces of length class c
 * (0: 17..32, 1: 33..64, 2: 65..128, 3: 129..256, 4: 257..1024, 5: 1025..4096, 6: 4097..32768, 7: longer bytes),
 * summed over chunks and devices, from the runs whose output the call returned; *lane_per_piece = 1 when the
 * lane-per-piece kernels merged them (largest rank 2^22 or above), 0 for the group and parallel-merge kernels.  After
 * a queued device series the counts describe its last call.  Reset to zeros where b200bpe_last_reruns is, and left at
 * zeros by a call that fails. */
int b200bpe_last_piece_classes(b200bpe_t *h, uint64_t *counts8, int *lane_per_piece);

/* Documents the most recent b200bpe_encode_bytes_batch call on this handle found not to be well-formed UTF-8 and
 * repaired, summed over chunks and devices.  0 after any other encode call and after a call that failed. */
int b200bpe_last_bytes_repairs(b200bpe_t *h, uint64_t *n_docs_repaired);

/* What the most recent b200bpe_encode_with_unstable_batch call on this handle did, summed over chunks and devices:
 * [0] documents with unstable bytes, [1] completion candidates encoded (run 2), [2] of those, the ones that took
 * byte_pair_encode (single-piece mode: not UTF-8, or the whitespace split), [3] candidate rounds, [4] completions
 * returned.  Reset to zeros where b200bpe_last_reruns is, and left at zeros by a call that fails. */
int b200bpe_last_unstable(b200bpe_t *h, uint64_t *stats5);

/* What the miss memo did in the most recent encode call on this handle, summed over chunks and devices, from the runs
 * whose output the call returned: *misses = pieces of up to 16 bytes that are not tokens (a single byte only when the
 * vocabulary lacks it), *merged = those merged (one per distinct piece, plus every piece of 16 bytes and every piece the
 * memo did not place), *unplaced = pieces of up to 15 bytes the memo did not place: they found neither their key nor an
 * empty slot within 8 probe steps, or their part of the memo had stopped (full, or too few repeats to pay).  The memo lives for one call; its size is
 * B200BPE_MISS_MEMO_SLOTS slots (0: off, every miss is merged) or, unset, one slot per 128 bytes of a chunk, from 2^12
 * to 2^21.  After a queued device series the counts describe its last call.  Reset to zeros where b200bpe_last_reruns
 * is, and left at zeros by a call that fails. */
int b200bpe_last_miss_memo(b200bpe_t *h, uint64_t *misses, uint64_t *merged, uint64_t *unplaced);

/* How the most recent host-buffer encode or count call on this handle cut documents larger than a chunk: *seams =
 * chunk boundaries placed inside documents, *docs_cut = documents with at least one of them.  Reset to zeros where
 * b200bpe_last_reruns is, and left at zeros by a call that fails. */
int b200bpe_last_doc_seams(b200bpe_t *h, uint64_t *seams, uint64_t *docs_cut);

/* Sizes of the device tables (bytes) for reporting: [0] piece tables (narrow + wide), [1] pair table,
 * [2] long-token table + blob, [3] Unicode class tables. */
int b200bpe_table_bytes(b200bpe_t *h, uint64_t *bytes4);

/* Number of CUDA devices the library can see (0 when there is none: every constructor then fails with
 * B200BPE_ECUDA -- there is no CPU fallback). */
int b200bpe_device_count(void);

const char *b200bpe_last_error(void);
const char *b200bpe_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200BPE_H */
