/* b2t.h -- C ABI of the CUDA (H100, sm_90a) batched tokenization engine (libb2t.so).
 *
 * Drop-in boundary for ONE path of huggingface/tokenizers: `Tokenizer::encode_batch` for ByteLevel-BPE
 * (GPT-2 / Llama-3 style) and Whitespace + WordPiece.  Each entry point names the reference interface it
 * replaces (paths relative to tokenizers/src of huggingface/tokenizers unless noted).  A Rust host would bind this file
 * with an `extern "C"` block (see INTEGRATION.md); the Python shim in tokenizers_b200/ binds it with ctypes.
 *
 * Conventions: plain pointers and sizes only; every function returns a b2t_status value (0 = ok) unless noted; the
 * message of the last error on the calling thread is available from b2t_last_error().  No CPU fallback exists:
 * configurations outside the supported set fail with B2T_ERR_UNSUPPORTED, and every encode entry point needs a
 * CUDA device (sm_90a).
 */
#ifndef B2T_H_
#define B2T_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2t_engine b2t_engine;
typedef struct b2t_result b2t_result;

typedef enum {
  B2T_OK = 0,
  B2T_ERR_INVALID = 1,     /* bad argument */
  B2T_ERR_UNSUPPORTED = 2, /* configuration outside the hot path (the reference would handle it on CPU) */
  B2T_ERR_CUDA = 3,        /* CUDA runtime error, message has the details */
  B2T_ERR_VOCAB = 4,       /* merge token out of vocabulary / missing [UNK] (models/bpe/mod.rs:12-36, wordpiece/mod.rs:17-22) */
  B2T_ERR_TOO_LARGE = 5,   /* batch exceeds the per-call device limits */
  B2T_ERR_TRUNCATION = 6   /* TruncationError::SequenceTooShort (utils/truncation.rs:155): a pair cannot be cut to max_length;
                              or, with overflowing parts, a sequence that has to be cut to a max_len no larger than the
                              stride (the reference panics there: tokenizer/encoding.rs:318) */
} b2t_status;

/* models::ModelWrapper variants on the path (models/mod.rs:60-68) */
typedef enum { B2T_MODEL_BPE = 0, B2T_MODEL_WORDPIECE = 1 } b2t_model_kind;

/* pre_tokenizers::PreTokenizerWrapper configurations on the path (pre_tokenizers/mod.rs:28-62) */
typedef enum {
  B2T_PRETOK_BYTELEVEL = 0,         /* ByteLevel{use_regex=true}: GPT-2 pattern, byte_level.rs:43-46,119-148 */
  B2T_PRETOK_LLAMA3 = 1,            /* Sequence[Split(tiktoken pattern, Isolated), ByteLevel{use_regex=false}] */
  B2T_PRETOK_WHITESPACE = 2,        /* Whitespace: whitespace.rs:20-29 */
  B2T_PRETOK_BYTELEVEL_NOREGEX = 3, /* ByteLevel{use_regex=false}: the whole sequence is one pre-token */
  B2T_PRETOK_BERT = 4               /* BertPreTokenizer: pre_tokenizers/bert.rs:5-19 (whitespace removed, punctuation isolated) */
} b2t_pretok_kind;

/* normalizers::BertNormalizer (normalizers/bert.rs:52-136), in front of a WordPiece pipeline: b2t_config.bert_normalizer =
 * B2T_NORM_BERT | the enabled steps (strip_accents: None resolves to lowercase, bert.rs:128).  The normalizer runs on the
 * device; offsets refer to the ORIGINAL text through the alignments (tokenizer/normalizer.rs:317-428).  0 = no normalizer. */
enum { B2T_NORM_BERT = 0x100, B2T_NORM_CLEAN_TEXT = 1, B2T_NORM_CHINESE_CHARS = 2, B2T_NORM_STRIP_ACCENTS = 4, B2T_NORM_LOWERCASE = 8 };

/* Engine configuration = what `TokenizerBuilder` (tokenizer/mod.rs:315-437) receives for this path:
 * BPE::builder().vocab_and_merges(..).ignore_merges(..) (models/bpe/model.rs:36-210) or
 * WordPiece::builder().vocab(..).unk_token(..).continuing_subword_prefix(..).max_input_chars_per_word(..)
 * (models/wordpiece/mod.rs:40-120), plus the pre-tokenizer flags. Strings are UTF-8, exactly as in tokenizer.json. */
typedef struct {
  uint32_t struct_size; /* sizeof(b2t_config), for ABI evolution */
  int32_t model;        /* b2t_model_kind */
  int32_t pretok;       /* b2t_pretok_kind */
  int32_t add_prefix_space; /* ByteLevel.add_prefix_space (byte_level.rs:57-68) */
  int32_t ignore_merges;    /* BPE.ignore_merges (models/bpe/model.rs:558-567) */
  /* vocabulary: n_vocab token strings, packed back to back; token i = vocab_bytes[vocab_off[i] .. vocab_off[i+1]) */
  uint32_t n_vocab;
  const uint8_t* vocab_bytes;
  const uint32_t* vocab_off; /* n_vocab + 1 */
  const uint32_t* vocab_ids; /* n_vocab */
  /* BPE merges in rank order: merge i = (string 2i, string 2i+1) of the packed list (models/bpe/model.rs:252-275) */
  uint32_t n_merges;
  const uint8_t* merge_bytes;
  const uint32_t* merge_off; /* 2 * n_merges + 1 */
  /* WordPiece */
  const char* unk_token;                 /* NUL-terminated, may be NULL for BPE */
  const char* continuing_subword_prefix; /* NUL-terminated, e.g. "##" */
  uint32_t max_input_chars_per_word;     /* 100 in bert */
  int32_t device;                        /* CUDA device ordinal, -1 = current device */
  int32_t bert_normalizer;               /* B2T_NORM_* flags, 0 = none */
} b2t_config;

/* encode flags */
enum {
  B2T_WANT_OFFSETS = 1u,   /* produce (start, end) per token */
  B2T_WANT_WORD_IDS = 2u,  /* produce the pre-token ordinal per token (Encoding.words, tokenizer/pre_tokenizer.rs:252-256) */
  B2T_OFFSETS_BYTES = 4u,  /* OffsetType::Byte (Rust encode_batch) instead of OffsetType::Char (encode_batch_char_offsets,
                              what the Python binding always uses: bindings/python/src/tokenizer.rs:1332) */
  B2T_NO_ADDED_TOKENS = 8u,   /* skip the added-token extraction of an engine that has added tokens (the caller knows the text
                                 holds none, or has split it already) */
  B2T_FLAG_ADDED_IDS = 16u    /* mark the tokens that come from the added vocabulary with bit 31 of their id */
};

/* AddedToken properties (tokenizer/added_vocabulary.rs:11-76) */
enum { B2T_ADDED_SINGLE_WORD = 1u, B2T_ADDED_LSTRIP = 2u, B2T_ADDED_RSTRIP = 4u, B2T_ADDED_NORMALIZED = 8u };

/* Replaces TokenizerBuilder::build for the path.  The tables are uploaded to the device once; the engine is
 * immutable afterwards and may be used from several host threads: every host-buffer call (b2t_encode_batch,
 * b2t_encode_batch_dense, b2t_encode_pairs_dense, b2t_pre_tokenize_batch) runs on device workspaces and streams of its own (up to four calls in
 * flight, further ones wait), so their copies and kernels overlap; the device-resident entry points share one workspace
 * (their result lives in it) and serialise.  With profiling on (b2t_engine_set_profiling) calls are meant to be made one at a time. */
int b2t_engine_create(const b2t_config* cfg, b2t_engine** out);
void b2t_engine_destroy(b2t_engine* e);

/* Replaces AddedVocabulary::add_tokens / refresh_added_tokens (tokenizer/added_vocabulary.rs:270-420) for the path: the
 * tokens the encode entry points extract from the text BEFORE pre-tokenization, like extract_and_normalize without a
 * normalizer (added_vocabulary.rs:523-564: non-normalized tokens first, then the normalized ones on the remaining pieces;
 * leftmost-longest, single_word / lstrip / rstrip).  Token i = bytes[off[i] .. off[i+1]), ids[i] < 2^20, flags[i] = OR of
 * B2T_ADDED_*.  The extraction runs on the device (no re-packing: span boundaries become hard boundaries of the scan, a
 * span becomes one pre-token that carries the token's id).  Not combinable with add_prefix_space (B2T_ERR_UNSUPPORTED); a
 * batch whose spans do not fit the device limits (a span over 256 bytes after lstrip / rstrip, more spans than one per
 * 16 input bytes, the reference's overlapping-span corner case) fails with B2T_ERR_UNSUPPORTED -- the host can then split
 * the text itself and pass B2T_NO_ADDED_TOKENS.  n_tokens = 0 clears the set.  Not to be called concurrently with encodes. */
int b2t_engine_set_added_tokens(b2t_engine* e, uint32_t n_tokens, const uint8_t* bytes, const uint32_t* off,
                                const uint32_t* ids, const uint8_t* flags);

/* Replaces TokenizerImpl::encode_batch / encode_batch_char_offsets / encode_batch_fast (tokenizer/mod.rs:1337-1401)
 * for raw (not pre-tokenized) single sequences with add_special_tokens=false.  HOST buffers: `bytes` holds the
 * documents back to back, document d = bytes[doc_off[d] .. doc_off[d+1]); doc_off[0] must be 0 and doc_off must be
 * non-decreasing (checked: B2T_ERR_INVALID otherwise -- nothing unordered reaches a kernel).  The call copies the
 * input to the device in chunks, runs the kernels and copies the token CSR back into pinned host memory owned by
 * the result.  flags = 0 is the encode_batch_fast analogue (ids only). */
int b2t_encode_batch(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, uint32_t flags,
                     b2t_result** out);

/* Same, with the packed batch already in device memory (d_bytes 16-byte aligned, n_bytes = doc_off[n_docs] < 2^31) and the
 * result left in device memory (owned by the engine, valid until the next call on this engine or b2t_result_free).
 * `stream` is a cudaStream_t (NULL = the engine's own stream); the call is asynchronous with respect to the host
 * except for one small device-to-host read of the token count.  This is the entry point the roofline numbers use. */
int b2t_encode_batch_device(b2t_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off,
                            uint32_t n_docs, uint32_t flags, void* stream, b2t_result** out);

/* The same call in two halves, for callers that place the result themselves -- the multi-GPU path: the reference fans a
 * batch out over rayon threads (tokenizer/mod.rs:1345-1348) and collects the encodings in input order; here every rank
 * (one process per GPU) encodes its contiguous shard of the batch and writes its part of the token CSR straight at its
 * displacement of the buffer that the all-gather then completes (tokenizers_b200/parallel.py encode_batch_sharded).
 *   begin : everything up to the token counts; *n_tokens = tokens of this shard (one small device-to-host read).
 *   finish: writes ids[0..n_tokens), offsets[0..2 n_tokens) (if requested at begin), word_ids (if requested) and
 *           row_ptr[0..n_docs] = token_base + the shard's row_ptr to the DEVICE pointers given (already displaced by
 *           the caller); asynchronous on `stream`.  No other call on this engine between begin and finish. */
int b2t_encode_batch_device_begin(b2t_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off,
                                  uint32_t n_docs, uint32_t flags, void* stream, uint64_t* n_tokens);
int b2t_encode_batch_device_finish(b2t_engine* e, uint32_t* d_ids, uint32_t* d_offsets, uint32_t* d_word_ids,
                                   uint64_t* d_row_ptr, uint64_t token_base, void* stream);

/* Dense mode: the steps the reference runs AFTER the path for a batch of single sequences -- truncation
 * (utils/truncation.rs:70-166, kept part of Encoding::truncate, tokenizer/encoding.rs:307-388), the special-token template
 * `pre $A post` (processors/template.rs:646-, BertProcessing / RobertaProcessing single form) and padding
 * (utils/padding.rs:50-81), as TokenizerImpl::post_process orders them (tokenizer/mod.rs:1265-1317) -- done on the device:
 * the result is a dense [n_docs, L] tensor of ids (+ attention mask + row lengths) instead of the token CSR, which never
 * leaves the device.  With B2T_DENSE_OVERFLOW the overflowing parts (stride) of a truncated sequence become rows of their own,
 * and with B2T_DENSE_OFFSETS the character offsets of every position come back too (see below). */
enum {
  B2T_DENSE_OVERFLOW = 1u,  /* return_overflowing_tokens: every part Encoding::truncate makes (tokenizer/encoding.rs:307-388) is a
                               row -- an input's kept row first, then its overflowing rows (`[e] + e.overflowing`), each with the
                               template around it; b2t_result_row_sample maps each row to its input */
  B2T_DENSE_OFFSETS = 2u,   /* return_offsets_mapping: [rows, L] (start, end) char offsets relative to the row's sequence
                               (growing_offsets = false), (0, 0) for special tokens and padding */
  B2T_DENSE_TRIM_OFFSETS = 4u,  /* trim_offsets (pre_tokenizers/byte_level.rs:202-234 process_offsets, on every part of every
                                   sequence): the offset rows skip a token's leading / trailing U+0120 or whitespace chars --
                                   of its vocabulary string, or for an added token of the span it matched.  Needs
                                   B2T_DENSE_OFFSETS (else B2T_ERR_INVALID) and a BPE engine (else B2T_ERR_UNSUPPORTED).  An
                                   added token with both lstrip and rstrip that absorbed whitespace in a row fails the call
                                   with B2T_ERR_UNSUPPORTED: which side the whitespace came from is not in its offsets. */
  B2T_DENSE_TRIM_PREFIX_SPACE = 8u,  /* the post-processor's add_prefix_space: a part's first token (or one at offset 0) keeps a
                                        single leading space.  Only with B2T_DENSE_TRIM_OFFSETS. */
  B2T_DENSE_SPECIAL_MASK = 16u,  /* special_tokens_mask: [rows, L] u8, 1 for template tokens and padding (encoding.rs:465-519) */
  B2T_DENSE_SEQUENCE_IDS = 32u,  /* sequence ids: [rows, L] i8, 0 for A's tokens, 1 for B's, -1 (None) for template tokens and
                                    padding (encoding.rs:137-145) */
  B2T_DENSE_WORD_IDS = 64u       /* word ids: [rows, L] u32, the word of every sequence token (restarting per sequence),
                                    0xFFFFFFFF (None) for template tokens and padding */
};
typedef struct {
  uint32_t struct_size;        /* sizeof(b2t_dense_spec) */
  uint32_t length;             /* PaddingStrategy::Fixed(length); 0 = BatchLongest (needs the batch in one device pass: < 2^31 bytes) */
  uint32_t pad_to_multiple_of; /* PaddingParams.pad_to_multiple_of, 0 = none */
  uint32_t max_length;         /* TruncationParams.max_length, special tokens included; 0 = no truncation */
  uint32_t pad_id;             /* PaddingParams.pad_id */
  int32_t truncate_left;       /* TruncationDirection::Left: keep the LAST tokens */
  int32_t pad_left;            /* PaddingDirection::Left */
  uint32_t n_pre, n_post;      /* special tokens of the single-sequence template before / after the sequence (<= 8 each) */
  const uint32_t* pre_ids;
  const uint32_t* post_ids;
  uint32_t want_mask;          /* also return the attention mask (u8 per position); row lengths always come back */
  /* appended fields: a struct_size that ends before them (the size of the struct without them) reads them as 0 */
  uint32_t stride;             /* TruncationParams.stride: tokens consecutive parts share (B2T_DENSE_OVERFLOW only) */
  uint32_t dense_flags;        /* B2T_DENSE_* */
} b2t_dense_spec;

/* HOST buffers in (as b2t_encode_batch), pinned host rows out.  A row that does not fit L (Fixed length without a
 * sufficient truncation; the reference returns a longer row there) fails the batch with B2T_ERR_INVALID.  With
 * B2T_DENSE_OVERFLOW, L is still the longest KEPT row under BatchLongest (pad_encodings looks at the top-level encodings
 * only), and an overflowing row longer than L fails the batch the same way (the reference returns it unpadded and longer:
 * a whole sequence overflows when it is cut to 0 tokens). */
int b2t_encode_batch_dense(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs,
                           const b2t_dense_spec* spec, b2t_result** out);
/* Device buffers in (as b2t_encode_batch_device), device rows out (owned by the engine until the next call). */
int b2t_encode_batch_dense_device(b2t_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off,
                                  uint32_t n_docs, const b2t_dense_spec* spec, void* stream, b2t_result** out);
/* Dense results: R rows (R = b2t_result_n_docs without B2T_DENSE_OVERFLOW); row d = ids[d * L .. (d + 1) * L);
 * row_lengths[d] = tokens of row d that are not padding.  b2t_result_n_docs stays the number of inputs. */
uint32_t b2t_result_dense_length(const b2t_result* r);        /* L */
uint32_t b2t_result_dense_rows(const b2t_result* r);          /* R (0 for a result that is not dense); R < 2^31, else the call
                                                                 fails with B2T_ERR_TOO_LARGE */
const uint32_t* b2t_result_dense_ids(const b2t_result* r);    /* R * L */
const uint8_t* b2t_result_attention_mask(const b2t_result* r); /* R * L, or NULL */
const uint32_t* b2t_result_row_lengths(const b2t_result* r);  /* R */
const uint32_t* b2t_result_row_sample(const b2t_result* r);   /* R: the input of each row (overflow_to_sample_mapping), or NULL
                                                                 without B2T_DENSE_OVERFLOW */
const uint32_t* b2t_result_dense_offsets(const b2t_result* r); /* R * L * 2 (start, end), or NULL without B2T_DENSE_OFFSETS */
const uint8_t* b2t_result_special_tokens_mask(const b2t_result* r); /* R * L, or NULL without B2T_DENSE_SPECIAL_MASK */
const int8_t* b2t_result_sequence_ids(const b2t_result* r);          /* R * L, or NULL without B2T_DENSE_SEQUENCE_IDS */
const uint32_t* b2t_result_dense_word_ids(const b2t_result* r);      /* R * L, or NULL without B2T_DENSE_WORD_IDS */

/* Dense mode for PAIRS of sequences (EncodeInput::Dual): what the reference runs after the path for a batch of pairs --
 * truncate_encodings with a pair (utils/truncation.rs:70-162, kept parts only), the pair template (processors/template.rs:
 * 544-643 apply_template; BertProcessing / RobertaProcessing pair forms; default_process without a post-processor) and
 * padding (utils/padding.rs:50-81), as TokenizerImpl::post_process orders them (tokenizer/mod.rs:1265-1317) -- done on the
 * device.  The batch is 2 n_pairs documents: document 2p is the first sequence of pair p, 2p + 1 the second.  The result
 * is n_pairs dense rows of ids, type ids (+ attention mask + row lengths); b2t_result_n_docs is n_pairs.  With
 * B2T_DENSE_OVERFLOW each sequence is cut with the max_len truncate_encodings gives it, and a pair whose sequences have
 * 1 + o_x and 1 + o_y parts (X / Y = first / second sequence in template order) gives (1 + o_x)(1 + o_y) rows in
 * Encoding::merge_with's order (tokenizer/encoding.rs:408-463): (0, 0); (i, 0), (i, 1) .. (i, o_y) for i = 1 .. o_x; then
 * (0, 1) .. (0, o_y).  A kept part takes its piece's type id, an overflowing part overflow_type_a / _b. */
enum { B2T_TRUNC_LONGEST_FIRST = 0, B2T_TRUNC_ONLY_FIRST = 1, B2T_TRUNC_ONLY_SECOND = 2 };  /* TruncationStrategy */
/* the sequence pieces of a template's piece list (token ids are < 2^20, so these never collide with one) */
enum { B2T_PIECE_A = 0x80000000u, B2T_PIECE_B = 0x80000001u };
typedef struct {
  uint32_t struct_size;        /* sizeof(b2t_pair_dense_spec) */
  uint32_t length;             /* PaddingStrategy::Fixed(length); 0 = BatchLongest (the batch in one device pass: < 2^31 bytes) */
  uint32_t pad_to_multiple_of; /* PaddingParams.pad_to_multiple_of, 0 = none */
  uint32_t max_length;         /* TruncationParams.max_length, special tokens included; 0 = no truncation */
  int32_t strategy;            /* B2T_TRUNC_* */
  int32_t truncate_left;       /* TruncationDirection::Left: keep the LAST tokens of each sequence */
  uint32_t pad_id;             /* PaddingParams.pad_id */
  uint32_t pad_type_id;        /* PaddingParams.pad_type_id (<= 255) */
  int32_t pad_left;            /* PaddingDirection::Left */
  /* the pair template (Template::pair, processors/template.rs): n_pieces entries, each a special token id or B2T_PIECE_A /
   * B2T_PIECE_B (exactly one of each, in the template's order), with its type id (<= 255).  Without a post-processor:
   * {A: 0, B: 1}; with add_special_tokens = false: the template's two sequence pieces only. At most 8 special tokens
   * before, between and after the sequences. */
  uint32_t n_pieces;
  const uint32_t* piece_ids;
  const uint32_t* piece_types;
  uint32_t want_mask;          /* also return the attention mask (u8 per position); type ids and row lengths always come back */
  /* appended fields: a struct_size that ends before them (the size of the struct without them) reads them as 0 */
  uint32_t stride;             /* TruncationParams.stride (B2T_DENSE_OVERFLOW only) */
  uint32_t dense_flags;        /* B2T_DENSE_* */
  uint32_t overflow_type_a;    /* type id of the overflowing parts of A / B (<= 255): the type id they had before the template, */
  uint32_t overflow_type_b;    /* 0 / 1 -- 0 / 0 under RobertaProcessing with special tokens (processors/roberta.rs) */
} b2t_pair_dense_spec;

/* HOST buffers in (doc_off holds 2 n_pairs + 1 offsets), pinned host rows out.  A pair that cannot be truncated fails the
 * batch with B2T_ERR_TRUNCATION; a row that does not fit a fixed length with B2T_ERR_INVALID (as b2t_encode_batch_dense). */
int b2t_encode_pairs_dense(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_pairs,
                           const b2t_pair_dense_spec* spec, b2t_result** out);
/* Device buffers in (as b2t_encode_batch_device, 2 n_pairs + 1 offsets), device rows out (owned by the engine until the next call). */
int b2t_encode_pairs_dense_device(b2t_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off,
                                  uint32_t n_pairs, const b2t_pair_dense_spec* spec, void* stream, b2t_result** out);
/* Encoding::get_type_ids of every row of a pair result: row p = type_ids[p * L .. (p + 1) * L); NULL for other results. */
const uint8_t* b2t_result_type_ids(const b2t_result* r);

/* Replaces PreTokenizer::pre_tokenize (tokenizer/mod.rs:65-67) for a batch: the splits of every document as
 * (start, end) BYTE offsets into the document (offsets[2k], offsets[2k+1]); row_ptr delimits documents.  ids and
 * word_ids are absent.  Host buffers in, pinned host buffers out.  The text as given is split: the engine's normalizer
 * and added tokens do not apply.  (With add_prefix_space the split that contains the inserted space starts at the
 * first byte of the document.) */
int b2t_pre_tokenize_batch(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs,
                           b2t_result** out);

/* Decoding (tokenizer/mod.rs:935-953 decode, :1404-1416 decode_batch): ids -> text on the device, for the decoders of the
 * pipelines the engine encodes.  Each id becomes the added vocabulary's string for it, else the model's; ids that are in
 * neither (ids at or above the largest id, 0xFFFFFFFF, ids with bit 31) are dropped; with B2T_DECODE_SKIP_SPECIAL a token
 * whose string is the content of a special added token is dropped.  The decoder then joins the kept tokens:
 *   B2T_DECODER_NONE      tokens.join(" ")
 *   B2T_DECODER_WORDPIECE decoders/wordpiece.rs:31-61: every kept token but the first loses `prefix` (or gains " "), then
 *                         the cleanup replacements run on that token alone
 *   B2T_DECODER_BYTELEVEL pre_tokenizers/byte_level.rs:156-171: chars -> bytes through the inverse byte map (a token with a
 *                         char outside it contributes its UTF-8), then String::from_utf8_lossy once per row */
typedef enum { B2T_DECODER_NONE = 0, B2T_DECODER_BYTELEVEL = 1, B2T_DECODER_WORDPIECE = 2 } b2t_decoder_kind;
enum { B2T_ADDED_SPECIAL = 16u };       /* b2t_decoder_spec.added_flags: AddedToken.special (with the B2T_ADDED_* bits) */
enum { B2T_DECODE_SKIP_SPECIAL = 1u };  /* decode flags: skip_special_tokens */
typedef struct {
  uint32_t struct_size;     /* sizeof(b2t_decoder_spec) */
  int32_t kind;             /* b2t_decoder_kind; any other value fails with B2T_ERR_UNSUPPORTED */
  const char* prefix;       /* WordPiece: NUL-terminated prefix ("##"); NULL = "" */
  int32_t cleanup;          /* WordPiece: cleanup */
  /* the whole added vocabulary (also on engines whose encode path does not extract it): token i = added_bytes[added_off[i]
   * .. added_off[i+1]) with id added_ids[i] (< 2^20) and flags added_flags[i] (B2T_ADDED_NORMALIZED, B2T_ADDED_SPECIAL) */
  uint32_t n_added;
  const uint8_t* added_bytes;
  const uint32_t* added_off;
  const uint32_t* added_ids;
  const uint8_t* added_flags;
} b2t_decoder_spec;

/* Sets the decoder of the engine's decode entry points (spec = NULL: none; the decode calls then fail with
 * B2T_ERR_INVALID).  Builds one table entry per id in [0, largest id] (ids < 2^20): whether the id exists, whether
 * skip_special_tokens drops it, and its image as the first kept token and as a later one.  Refused with
 * B2T_ERR_UNSUPPORTED (the engine keeps no decoder; encoding is unaffected): an unknown kind, added tokens with
 * normalized=true on an engine with a normalizer (the reference's tree and its release disagree on their string), an
 * image over 16383 bytes.  Not to be called concurrently with decodes. */
int b2t_engine_set_decoder(b2t_engine* e, const b2t_decoder_spec* spec);

/* The table b2t_engine_set_decoder builds and the kernels read, from the configuration's vocabulary and the spec alone
 * (host only, no device needed).  Entry id = table[id]: bits 0-31 the image's offset in pool, bits 32-45 the first
 * image's length, bits 46-59 the later image's length (its bytes follow the first image's), bit 60 the id exists, bit 61
 * skip_special_tokens drops it.  Call with table = pool = NULL for *n_ids and *pool_bytes, then with buffers that large. */
int b2t_decoder_images(const b2t_config* cfg, const b2t_decoder_spec* spec, uint64_t* table, uint8_t* pool, uint32_t* n_ids,
                       uint64_t* pool_bytes);

/* Decodes n_rows rows of ids: row r = ids[row_ptr[r] .. row_len ? row_ptr[r] + row_len[r] : row_ptr[r+1]) -- the token CSR
 * of b2t_encode_batch (row_len = NULL), or padded [n, L] rows with their lengths (row_ptr[r] = r L).  row_ptr must be
 * non-decreasing and every row inside [0, n_ids) (B2T_ERR_INVALID otherwise).  Result: the UTF-8 text of every row back to
 * back, row r = text[text_off[r] .. text_off[r+1]) (b2t_result_text / b2t_result_text_off; b2t_result_n_docs = n_rows,
 * b2t_result_n_tokens = text_off[n_rows]), exactly decode(row, skip_special_tokens).  Per-call limits (B2T_ERR_TOO_LARGE):
 * n_ids < 2^31, the images of one row (its text before the lossy step) below 2^30 bytes.  HOST buffers in, pinned host text out; the call runs in chunks of
 * whole rows on a slot set of its own, as b2t_encode_batch does (a row larger than a chunk is a chunk of its own), and
 * concurrently with other host calls.  Within the call only a chunk's copy of its text back overlaps the next chunk: each
 * chunk waits for the host to read its text size (and for ByteLevel whether the lossy rewrite runs) before its text is
 * written. */
int b2t_decode_batch(b2t_engine* e, const uint32_t* ids, uint64_t n_ids, const uint64_t* row_ptr, const uint32_t* row_len, uint32_t n_rows,
                     uint32_t flags, b2t_result** out);
/* Device buffers in, device text out (owned by the engine, valid until the next device-resident call), on `stream`. */
int b2t_decode_batch_device(b2t_engine* e, const uint32_t* d_ids, uint64_t n_ids, const uint64_t* d_row_ptr, const uint32_t* d_row_len,
                            uint32_t n_rows, uint32_t flags, void* stream, b2t_result** out);
const uint8_t* b2t_result_text(const b2t_result* r);       /* text_off[n_rows] bytes, NULL for results that are not decodes */
const uint64_t* b2t_result_text_off(const b2t_result* r);  /* n_rows + 1, NULL for results that are not decodes */

/* Result accessors (Encoding fields of tokenizer/encoding.rs:11-31 as one CSR over the batch).  Pointers are host
 * pointers for b2t_encode_batch / b2t_pre_tokenize_batch and device pointers for b2t_encode_batch_device. */
uint64_t b2t_result_n_tokens(const b2t_result* r);
uint32_t b2t_result_n_docs(const b2t_result* r);
int b2t_result_on_device(const b2t_result* r);
const uint32_t* b2t_result_ids(const b2t_result* r);      /* n_tokens */
const uint32_t* b2t_result_offsets(const b2t_result* r);  /* 2 * n_tokens, or NULL */
const uint32_t* b2t_result_word_ids(const b2t_result* r); /* n_tokens, or NULL */
const uint64_t* b2t_result_row_ptr(const b2t_result* r);  /* n_docs + 1 */
/* Host results return their pinned buffers to the engine's pool: free every result BEFORE b2t_engine_destroy. */
void b2t_result_free(b2t_result* r);

/* Pinned host memory for callers that want b2t_encode_batch to copy straight from their buffer. */
int b2t_host_alloc(size_t bytes, void** out);
void b2t_host_free(void* p);

/* Per-kernel device timings of the last b2t_encode_batch_device call when profiling is on (CUDA events on the
 * launch stream).  names/ms arrays of capacity cap; returns the number of kernels launched by that call. */
int b2t_engine_set_profiling(b2t_engine* e, int on);
int b2t_engine_last_kernels(const b2t_engine* e, const char** names, float* ms, int cap);

/* Unicode class tables the scan kernels use, one byte per code point (0x110000 entries):
 * scheme 0 (Oniguruma: ByteLevel / Split): 1 = \p{L}, 2 = \p{N}, 3 = \s, 0 = other;
 * scheme 1 (Rust regex: Whitespace):       1 = \w, 3 = \s, 0 = other;
 * scheme 2 (BertPreTokenizer):              1 = word character, 3 = whitespace (removed), 0 = punctuation (isolated).
 * Host only, no device needed. */
int b2t_unicode_class_table(int scheme, uint8_t* out);

/* The BertNormalizer table the device kernels use, for inspection (host only, no device needed): the UTF-8 image of every
 * code point under `flags` (B2T_NORM_* steps), images back to back in `pool` (capacity `cap`, 5 MB is enough), code point c =
 * pool[off[c] .. off[c+1]) with off holding 0x110001 entries; an empty image = the character is dropped. */
int b2t_bert_normalizer_images(int32_t flags, uint8_t* pool, size_t cap, uint32_t* off);

/* Thread-local message of the last failing call. */
const char* b2t_last_error(void);
/* Library version string. */
const char* b2t_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B2T_H_ */
