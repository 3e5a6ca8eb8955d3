// dense_kernels.cuh -- the post-path steps of a single-sequence batch on the device: special-token template, truncation
// and padding, emitted as dense [n_docs, L] id / attention-mask tensors straight from the token CSR.
//
// Replaces, for batches of single sequences (paths relative to tokenizers/src of huggingface/tokenizers):
//   tokenizer/mod.rs:1265-1317       TokenizerImpl::post_process: truncate to max_length - n_added_tokens, template, padding
//   utils/truncation.rs:70-166       truncate_encodings, single sequence: keep the first (direction right) or the last
//                                    (direction left) max_length tokens -- the kept part of Encoding::truncate
//                                    (tokenizer/encoding.rs:307-388); with overflowing parts, every part is a row (below)
//   processors/template.rs:646-      apply_template for `pre $A post`: special tokens before / after the sequence
//   utils/padding.rs:50-81           pad_encodings: pad id on the right or left up to the common length, attention mask 0
// The CSR never leaves the device in this mode: a row costs L * 4 (+ L) bytes of D2H whatever the template holds.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2t {

constexpr int DENSE_MAX_SPECIAL = 8;
constexpr uint32_t DENSE_NO_LIMIT = 0xFFFFFFFFu;

struct DenseSpec {
  uint32_t L;          // row length of the output
  uint32_t keep_max;   // most tokens of the sequence itself that a row keeps (max_length - n_pre - n_post), DENSE_NO_LIMIT = no truncation
  uint32_t pad_id;
  uint32_t n_pre, n_post;
  int32_t trunc_left, pad_left;
  uint32_t pre[DENSE_MAX_SPECIAL], post[DENSE_MAX_SPECIAL];
};

// longest row (template included, after truncation) of the CSR -> *max_len (atomicMax; zeroed by the caller)
__global__ void row_len_max_kernel(const uint64_t* __restrict__ row_ptr, uint32_t n_docs, uint32_t keep_max, uint32_t n_special,
                                   uint32_t* __restrict__ max_len) {
  const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t len = 0;
  if (d < n_docs) {
    const uint64_t c = row_ptr[d + 1] - row_ptr[d];
    len = (uint32_t)(c < keep_max ? c : keep_max) + n_special;
  }
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) len = max(len, __shfl_xor_sync(0xFFFFFFFFu, len, s));
  if ((threadIdx.x & 31) == 0 && len) atomicMax(max_len, len);
}

// ---------------------------------------------------------------------------------------------------- overflow
// Overflowing parts (stride), for single sequences and pairs: Encoding::truncate (tokenizer/encoding.rs:307-388) splits a
// sequence of n tokens cut to max_len m into the kept part and its overflowing parts, consecutive parts sharing `stride`
// tokens; Encoding::merge_with (encoding.rs:408-463) combines the parts of a pair's two sequences.  Every part becomes a
// dense row of its own, with the template around it.
enum { ERR_STRIDE = 64u };   // ctl err bit: the reference panics, "`stride` must be strictly less than `max_len`" (encoding.rs:318)

// parts of a sequence of n tokens truncated to m with stride s (kept part included); 0 = the reference panics (s >= m
// while the sequence has to be cut to m > 0).  m = 0 keeps an empty part, the whole sequence is one overflowing part.
__host__ __device__ inline uint32_t seq_parts(uint32_t n, uint32_t m, uint32_t s) {
  if (n <= m) return 1;
  if (m == 0) return 2;
  if (s >= m) return 0;
  const uint32_t step = m - s;
  return 1 + (n - m + step - 1) / step;
}

// part k (0 = kept) of that sequence -> tokens [*first, *first + *len); direction left counts the parts from the end
__host__ __device__ inline void seq_part(uint32_t n, uint32_t m, uint32_t s, bool left, uint32_t k, uint32_t* first, uint32_t* len) {
  if (n <= m) { *first = 0; *len = n; return; }
  if (m == 0) { *first = 0; *len = k ? n : 0u; return; }
  const uint32_t off = k * (m - s);   // (< n for every part k)
  if (!left) { *first = off; *len = n - off > m ? m : n - off; return; }
  const uint32_t stop = n - off;
  *first = stop > m ? stop - m : 0u; *len = stop - *first;
}

// the longest part of that sequence (the rows' widths): the kept part when it is all, else m (or n when m = 0)
__host__ __device__ inline uint32_t seq_part_max(uint32_t n, uint32_t m, uint32_t parts) { return parts > 1 && m ? m : n; }

// row r of a pair whose first sequence in template order (X) has ox overflowing parts and the second (Y) oy -> the part
// (*i of X, *j of Y) it merges.  merge_with's order: (0, 0); then (i, 0), (i, 1) .. (i, oy) for i = 1 .. ox; then
// (0, 1) .. (0, oy).  32-bit arithmetic: the pair's rows, (1 + ox)(1 + oy), are fewer than 2^31.
__host__ __device__ inline void pair_row_part(uint32_t r, uint32_t ox, uint32_t oy, uint32_t* i, uint32_t* j) {
  if (r == 0) { *i = 0; *j = 0; return; }
  const uint32_t q = r - 1, w = oy + 1;
  if (q < ox * w) { *i = 1 + q / w; *j = q % w; return; }
  *i = 0; *j = 1 + (q - ox * w);
}

// What the overflow (and offset) instantiations of the row kernels read besides the spec.  Row d copies input
// row_sample[d] - sample_base, whose first row is row_base[that input].
struct DenseOverflow {
  const uint32_t* row_sample; const uint32_t* row_base;
  uint32_t sample_base, stride;
  uint32_t type_ox, type_oy;     // pairs: type ids of the overflowing parts of X / Y
  const uint2* offsets;          // the CSR's (start, end) per token (offset rows)
  uint2* out_off;                // [rows, L] offsets, (0, 0) for special tokens and padding
};

// ------------------------------------------------------------------------------------------------- row metadata
// The per-position fields of the reference's post-processed Encoding besides ids, type ids and offsets: the special-tokens
// mask (encoding.rs:465-519: 1 for template tokens and padding), sequence ids (encoding.rs:137-145: None for those, A's
// tokens 0 and B's 1 whatever the template order), word ids (the CSR's, None for those) -- and offset trimming:
//   pre_tokenizers/byte_level.rs:202-234  process_offsets, run on every part of every sequence after truncation and before
//                                         the template (roberta.rs:71-79, byte_level.rs:180-193)
enum { ERR_TRIM_AMBIGUOUS = 128u };   // ctl err bit: an lstrip + rstrip added token absorbed whitespace (added_trim_counts)
enum { TRIM_ALL_SPACE = 1u, TRIM_LSTRIP = 2u, TRIM_RSTRIP = 4u };

// process_offsets on one token's offsets o: ld / tr = its leading / trailing chars that are U+0120 or whitespace.  The
// start moves past ld, except that with the post-processor's add_prefix_space (aps) a first token of its part (`first`)
// or one at offset 0 keeps a single leading space; the end moves back by tr where o1 >= tr, never before the new start.
__host__ __device__ inline uint2 trim_span(uint2 o, uint32_t ld, uint32_t tr, bool first, bool aps) {
  const bool keep = (first || o.x == 0u) && aps && ld == 1u;
  const uint32_t n0 = ld > 0u && !keep ? (o.x + ld < o.y ? o.x + ld : o.y) : o.x;
  const uint32_t n1 = tr > 0u && o.y >= tr ? (o.y - tr > n0 ? o.y - tr : n0) : o.y;
  return make_uint2(n0, n1);
}

// An added token as process_offsets sees it: its text is the span it matched, content plus the whitespace lstrip / rstrip
// absorbed (tokenizer.py _span_spaces).  counts = leading | trailing << 16 whitespace-or-U+0120 chars of the content.
struct AddedTrim { uint32_t id, chars, counts, flags; };   // flags: TRIM_*

// The counts of an occurrence whose span is S chars long (o1 - o0).  The S - chars absorbed chars lie left of the content
// for lstrip alone, right of it for rstrip alone.  false: both flags and S > chars -- how the absorbed whitespace splits
// between the two sides is not in the offsets.
__host__ __device__ inline bool added_trim_counts(uint32_t S, const AddedTrim& a, uint32_t* ld, uint32_t* tr) {
  const bool l = (a.flags & TRIM_LSTRIP) != 0u, r = (a.flags & TRIM_RSTRIP) != 0u;
  const uint32_t extra = S > a.chars ? S - a.chars : 0u;
  if (l && r && extra) return false;
  if (a.flags & TRIM_ALL_SPACE) { *ld = S; *tr = S; return true; }
  *ld = (l ? extra : 0u) + (a.counts & 0xFFFFu);
  *tr = (r ? extra : 0u) + (a.counts >> 16);
  return true;
}

// What the META instantiations of the row kernels read and write besides the spec.  Null output = not asked for.
struct DenseMeta {
  const uint32_t* trim_vocab;    // per vocabulary id: leading | trailing << 16 whitespace-or-U+0120 chars; null = no trimming
  const AddedTrim* trim_added;   // the added tokens by ascending id (their CSR ids carry bit 31)
  uint32_t n_added, aps;         // aps: the post-processor's add_prefix_space
  const uint32_t* word_ids;      // the CSR's word ids (out_word)
  uint8_t* out_special; int8_t* out_seq; uint32_t* out_word;   // [rows, L]
  uint32_t* err;                 // ERR_TRIM_AMBIGUOUS, ERR_INTERNAL_META
};
enum { ERR_INTERNAL_META = 4u };   // (long_kernels.cuh ERR_INTERNAL: a marked id that is no added token)

// the offsets of sequence token `id` (a CSR id: bit 31 = added token), trimmed when M asks for it
__device__ __forceinline__ uint2 meta_offsets(const DenseMeta& M, uint32_t id, uint2 o, bool first) {
  if (!M.trim_vocab) return o;
  uint32_t ld, tr;
  if (id >> 31) {
    uint32_t lo = 0, hi = M.n_added;
    const uint32_t want = id & 0x7FFFFFFFu;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (M.trim_added[mid].id < want) lo = mid + 1; else hi = mid; }
    if (lo == M.n_added || M.trim_added[lo].id != want) { atomicOr(M.err, (unsigned)ERR_INTERNAL_META); return o; }
    if (!added_trim_counts(o.y - o.x, M.trim_added[lo], &ld, &tr)) { atomicOr(M.err, (unsigned)ERR_TRIM_AMBIGUOUS); return o; }
  } else {
    const uint32_t c = M.trim_vocab[id];
    ld = c & 0xFFFFu; tr = c >> 16;
  }
  return trim_span(o, ld, tr, first, M.aps != 0u);
}

// cell `cell` of the metadata rows: a sequence token of sequence `seq` at CSR position t, or (tok false) a template token
// or padding
__device__ __forceinline__ void meta_write(const DenseMeta& M, size_t cell, bool tok, uint32_t seq, uint64_t t) {
  if (M.out_special) M.out_special[cell] = tok ? 0 : 1;
  if (M.out_seq) M.out_seq[cell] = tok ? (int8_t)seq : (int8_t)-1;
  if (M.out_word) M.out_word[cell] = tok ? M.word_ids[t] : 0xFFFFFFFFu;
}

// One warp per row.  row_ptr is the (chunk-relative) CSR of `ids`; rows are written at out_* + d * L.
// A row that does not fit L (padding to a fixed length without truncation) raises bit 0 of *err and is cut -- the host
// turns that into an error, the reference would return a longer row there.
// OVER: n_docs counts rows, each the template around one part of its input (the host has checked that every row fits
// L); OFFS: the offset rows as well; META: the rows of DenseMeta (trimmed offsets, ids without the added-token mark), the
// part's first token at position n_pre.
template <bool OVER = false, bool OFFS = false, bool META = false>
__global__ void dense_rows_kernel(const uint32_t* __restrict__ ids, const uint64_t* __restrict__ row_ptr, uint32_t n_docs, const DenseSpec S,
                                  uint32_t* __restrict__ out_ids, uint8_t* __restrict__ out_mask, uint32_t* __restrict__ out_len,
                                  uint32_t* __restrict__ err, const DenseOverflow O = DenseOverflow{}, const DenseMeta M = DenseMeta{}) {
  const uint32_t d = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (d >= n_docs) return;
  uint32_t doc = d, first = 0;
  if constexpr (OVER) doc = O.row_sample[d] - O.sample_base;
  const uint64_t a = row_ptr[doc], cnt = row_ptr[doc + 1] - a;
  uint32_t keep = (uint32_t)(cnt < (uint64_t)S.keep_max ? cnt : (uint64_t)S.keep_max);
  if constexpr (OVER) seq_part((uint32_t)cnt, S.keep_max, O.stride, S.trunc_left, d - O.row_base[doc], &first, &keep);
  uint32_t len = S.n_pre + keep + S.n_post;
  if (len > S.L) {
    if (lane == 0 && err) atomicOr(err, 1u);
    keep = S.L > S.n_pre + S.n_post ? S.L - S.n_pre - S.n_post : 0u;
    len = S.n_pre + keep + S.n_post;
    if (len > S.L) return;
  }
  const uint64_t src = OVER ? a + first : a + (S.trunc_left ? cnt - keep : 0ull);
  const uint32_t start = S.pad_left ? S.L - len : 0u;
  uint32_t* const row = out_ids + (size_t)d * S.L;
  uint8_t* const mrow = out_mask ? out_mask + (size_t)d * S.L : nullptr;
  for (uint32_t j = lane; j < S.L; j += 32) {
    const uint32_t k = j - start;   // wraps below start: k >= len
    uint32_t v = S.pad_id;
    if (k < len) {
      if (k < S.n_pre) v = S.pre[k];
      else if (k < S.n_pre + keep) v = ids[src + (k - S.n_pre)];
      else v = S.post[k - S.n_pre - keep];
    }
    if constexpr (META) {
      const bool tok = k >= S.n_pre && k < S.n_pre + keep;
      const uint64_t t = src + (k - S.n_pre);
      uint2 o = make_uint2(0u, 0u);
      if (tok) {
        if constexpr (OFFS) o = meta_offsets(M, v, O.offsets[t], k == S.n_pre);
        v &= 0x7FFFFFFFu;
      }
      row[j] = v;
      if (mrow) mrow[j] = k < len ? 1 : 0;
      if constexpr (OFFS) O.out_off[(size_t)d * S.L + j] = o;
      meta_write(M, (size_t)d * S.L + j, tok, 0u, t);
    } else {
      row[j] = v;
      if (mrow) mrow[j] = k < len ? 1 : 0;
      if constexpr (OFFS) O.out_off[(size_t)d * S.L + j] = k >= S.n_pre && k < S.n_pre + keep ? O.offsets[src + (k - S.n_pre)] : make_uint2(0u, 0u);
    }
  }
  if (lane == 0 && out_len) out_len[d] = len;
}

// ---------------------------------------------------------------------------------------------------------- pairs
// A batch of pairs is a batch of 2n documents: document 2p is the first sequence (A) of pair p, 2p + 1 the second (B).
// Replaces, for such batches:
//   tokenizer/mod.rs:1272-1283       the pair is truncated to max_length - the special tokens of the pair template
//   utils/truncation.rs:70-162       truncate_encodings with a pair: budget 0, longest_first, only_first / only_second
//                                    (kept parts only, Encoding::truncate, tokenizer/encoding.rs:307-388)
//   processors/template.rs:544-643   apply_template for the pair: pre X mid Y post, X / Y = A / B in template order, every
//                                    token carrying its piece's type id (bert.rs, roberta.rs are such templates)
//   utils/padding.rs:50-81           pad_encodings: pad id, pad type id, attention mask 0
enum { ERR_TRUNCATION = 32u };   // ctl err bit: TruncationError::SequenceTooShort (utils/truncation.rs:155)
enum { PAIR_LONGEST_FIRST = 0u, PAIR_ONLY_FIRST = 1u, PAIR_ONLY_SECOND = 2u };

// truncate_encodings (utils/truncation.rs:70-162) on the lengths of a pair: n1, n2 tokens, `budget` tokens for both
// (DENSE_NO_LIMIT = no truncation) -> kept lengths *k1, *k2; false = SequenceTooShort, which fails the batch
__host__ __device__ inline bool pair_keep(uint32_t n1, uint32_t n2, uint32_t budget, uint32_t strategy, uint32_t* k1, uint32_t* k2) {
  *k1 = n1; *k2 = n2;
  if (budget == 0) { *k1 = 0; *k2 = 0; return true; }   // both sequences are cut to nothing, whatever the strategy
  if (n1 + n2 <= budget) return true;
  if (strategy == PAIR_LONGEST_FIRST) {
    const bool swap = n1 > n2;
    uint32_t a = swap ? n2 : n1;   // the shorter one
    uint32_t b = a > budget ? a : (a > budget - a ? a : budget - a);
    if (a + b > budget) { a = budget / 2; b = a + budget % 2; }
    if (swap) { const uint32_t t = a; a = b; b = t; }
    *k1 = n1 < a ? n1 : a; *k2 = n2 < b ? n2 : b;   // Encoding::truncate never lengthens
    return true;
  }
  const uint32_t to_remove = n1 + n2 - budget;
  uint32_t* const k = strategy == PAIR_ONLY_FIRST ? k1 : k2;
  if (*k > to_remove) { *k -= to_remove; return true; }
  return false;
}

struct PairDenseSpec {
  uint32_t L;            // row length of the output
  uint32_t budget;       // tokens A and B keep together (max_length - specials), DENSE_NO_LIMIT = no truncation
  uint32_t strategy;     // PAIR_*
  uint32_t pad_id, pad_type;
  int32_t trunc_left, pad_left;
  uint32_t b_first;      // 1: the template holds B before A (X = B, Y = A)
  uint32_t type_x, type_y;
  uint32_t n_pre, n_mid, n_post;
  uint32_t special[3 * DENSE_MAX_SPECIAL];   // pre, mid, post back to back: id | type id << 24
};

// longest pair row (template included, after truncation) -> *max_len (atomicMax; zeroed by the caller); a pair that
// cannot be truncated to the budget raises ERR_TRUNCATION in *err
__global__ void pair_len_max_kernel(const uint64_t* __restrict__ row_ptr, uint32_t n_pairs, uint32_t budget, uint32_t strategy,
                                    uint32_t n_special, uint32_t* __restrict__ max_len, uint32_t* __restrict__ err) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t len = 0;
  if (p < n_pairs) {
    const uint64_t a = row_ptr[2 * p], b = row_ptr[2 * p + 1], c = row_ptr[2 * p + 2];
    uint32_t k1, k2;
    if (!pair_keep((uint32_t)(b - a), (uint32_t)(c - b), budget, strategy, &k1, &k2)) atomicOr(err, ERR_TRUNCATION);
    len = k1 + k2 + n_special;
  }
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) len = max(len, __shfl_xor_sync(0xFFFFFFFFu, len, s));
  if ((threadIdx.x & 31) == 0 && len) atomicMax(max_len, len);
}

// One warp per pair.  row_ptr is the (chunk-relative) CSR of `ids` over the pair's two documents; rows are written at
// out_* + p * L.  A row that does not fit L is left unwritten: the host has found it through pair_len_max_kernel and
// fails the batch.  The spec is read in place (__grid_constant__), so the special-token look-up needs no local copy.
// OVER: one warp per row, row p merging part i of X with part j of Y (pair_row_part) -- a kept part takes its piece's
// type id, an overflowing one O.type_ox / O.type_oy; OFFS: the offset rows as well; META: the rows of DenseMeta, X's and
// Y's parts each with its own first token (positions e0 and e2), X's tokens of sequence b_first and Y's of the other.
template <bool OVER = false, bool OFFS = false, bool META = false>
__global__ void dense_pair_rows_kernel(const uint32_t* __restrict__ ids, const uint64_t* __restrict__ row_ptr, uint32_t n_pairs,
                                       const __grid_constant__ PairDenseSpec S, uint32_t* __restrict__ out_ids, uint8_t* __restrict__ out_type,
                                       uint8_t* __restrict__ out_mask, uint32_t* __restrict__ out_len, const __grid_constant__ DenseOverflow O = DenseOverflow{},
                                       const __grid_constant__ DenseMeta M = DenseMeta{}) {
  const uint32_t p = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= n_pairs) return;
  uint32_t q = p;
  if constexpr (OVER) q = O.row_sample[p] - O.sample_base;
  const uint64_t a = row_ptr[2 * q], b = row_ptr[2 * q + 1], c = row_ptr[2 * q + 2];
  const uint32_t n1 = (uint32_t)(b - a), n2 = (uint32_t)(c - b);
  uint32_t k1, k2;
  pair_keep(n1, n2, S.budget, S.strategy, &k1, &k2);   // (a SequenceTooShort pair fails the batch: its row does not matter)
  uint64_t src_x, src_y;
  uint32_t kx, ky, type_x = S.type_x, type_y = S.type_y;
  if constexpr (OVER) {   // each sequence is cut to its kept length (its own max_len): parts of X by parts of Y
    const uint32_t nx = S.b_first ? n2 : n1, ny = S.b_first ? n1 : n2, mx = S.b_first ? k2 : k1, my = S.b_first ? k1 : k2;
    uint32_t i, j, fx, fy;
    pair_row_part(p - O.row_base[q], seq_parts(nx, mx, O.stride) - 1, seq_parts(ny, my, O.stride) - 1, &i, &j);
    seq_part(nx, mx, O.stride, S.trunc_left, i, &fx, &kx);
    seq_part(ny, my, O.stride, S.trunc_left, j, &fy, &ky);
    src_x = (S.b_first ? b : a) + fx; src_y = (S.b_first ? a : b) + fy;
    if (i) type_x = O.type_ox;
    if (j) type_y = O.type_oy;
  } else {
    const uint64_t src1 = a + (S.trunc_left ? n1 - k1 : 0u), src2 = b + (S.trunc_left ? n2 - k2 : 0u);
    src_x = S.b_first ? src2 : src1; src_y = S.b_first ? src1 : src2;
    kx = S.b_first ? k2 : k1; ky = S.b_first ? k1 : k2;
  }
  // segment ends: pre | X | mid | Y | post
  const uint32_t e0 = S.n_pre, e1 = e0 + kx, e2 = e1 + S.n_mid, e3 = e2 + ky, len = e3 + S.n_post;
  if (len > S.L) return;
  const uint32_t start = S.pad_left ? S.L - len : 0u;
  uint32_t* const row = out_ids + (size_t)p * S.L;
  uint8_t* const trow = out_type + (size_t)p * S.L;
  uint8_t* const mrow = out_mask ? out_mask + (size_t)p * S.L : nullptr;
  for (uint32_t j = lane; j < S.L; j += 32) {
    const uint32_t k = j - start;   // wraps below start: k >= len
    uint32_t v = S.pad_id, t = S.pad_type;
    uint2 o = make_uint2(0u, 0u);
    if (k < e0 || (k >= e1 && k < e2) || (k >= e3 && k < len)) {
      const uint32_t s = S.special[k < e0 ? k : (k < e2 ? e0 + (k - e1) : e0 + S.n_mid + (k - e3))];
      v = s & 0xFFFFFFu; t = s >> 24;
    } else if (k < e1) {
      v = ids[src_x + (k - e0)]; t = type_x;
      if constexpr (OFFS) o = O.offsets[src_x + (k - e0)];
    } else if (k < e3) {
      v = ids[src_y + (k - e2)]; t = type_y;
      if constexpr (OFFS) o = O.offsets[src_y + (k - e2)];
    }
    if constexpr (META) {
      const bool in_x = k >= e0 && k < e1, tok = in_x || (k >= e2 && k < e3);
      const uint64_t at = in_x ? src_x + (k - e0) : src_y + (k - e2);
      if (tok) {
        if constexpr (OFFS) o = meta_offsets(M, v, o, k == (in_x ? e0 : e2));
        v &= 0x7FFFFFFFu;
      }
      meta_write(M, (size_t)p * S.L + j, tok, in_x == (S.b_first != 0u) ? 1u : 0u, at);
    }
    row[j] = v;
    trow[j] = (uint8_t)t;
    if (mrow) mrow[j] = k < len ? 1 : 0;
    if constexpr (OFFS) O.out_off[(size_t)p * S.L + j] = o;
  }
  if (lane == 0) out_len[p] = len;
}

// Count pass of the overflow rows: one thread per input (pairs: documents 2p, 2p + 1; single sequences: document p, cut
// to `budget` = keep_max).  -> row_count[p] = its rows; *max_all = the longest of ALL rows (template included, atomicMax;
// zeroed by the caller).  Raises ERR_TRUNCATION (SequenceTooShort, pairs) and ERR_STRIDE (the reference's stride panic;
// *stride_m = the largest max_len it panicked on) in *err.
__global__ void dense_count_kernel(const uint64_t* __restrict__ row_ptr, uint32_t n_inputs, uint32_t pairs, uint32_t budget, uint32_t strategy,
                                   uint32_t stride, uint32_t n_special, uint32_t* __restrict__ row_count, uint32_t* __restrict__ max_all,
                                   uint32_t* __restrict__ err, uint32_t* __restrict__ stride_m) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t len = 0;
  if (p < n_inputs) {
    uint32_t n1, n2 = 0, m1, m2 = 0;
    if (pairs) {
      const uint64_t a = row_ptr[2 * p], b = row_ptr[2 * p + 1], c = row_ptr[2 * p + 2];
      n1 = (uint32_t)(b - a); n2 = (uint32_t)(c - b);
      if (!pair_keep(n1, n2, budget, strategy, &m1, &m2)) atomicOr(err, ERR_TRUNCATION);
    } else {
      n1 = (uint32_t)(row_ptr[p + 1] - row_ptr[p]); m1 = budget;
    }
    uint32_t p1 = seq_parts(n1, m1, stride), p2 = seq_parts(n2, m2, stride);
    if (!p1 || !p2) {
      atomicOr(err, ERR_STRIDE);
      atomicMax(stride_m, !p1 ? m1 : m2);
      p1 = p2 = 1;
    }
    const uint64_t rows = (uint64_t)p1 * p2;
    row_count[p] = rows < 0x80000000ull ? (uint32_t)rows : 0x80000000u;   // (a sum of 2^31 or more fails the batch)
    len = n_special + seq_part_max(n1, m1, p1) + seq_part_max(n2, m2, p2);
  }
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) len = max(len, __shfl_xor_sync(0xFFFFFFFFu, len, s));
  if ((threadIdx.x & 31) == 0 && len) atomicMax(max_all, len);
}

// One warp per input: row_base[p] = its first row (the exclusive scan of row_count: local_excl + block_excl of a two-level
// scan over blocks of scan_block), row_sample[its rows] = p + sample_base (the input's index in the whole batch).
__global__ void dense_row_sample_kernel(const uint32_t* __restrict__ row_count, const unsigned long long* __restrict__ local_excl,
                                        const unsigned long long* __restrict__ block_excl, uint32_t scan_block, uint32_t n_inputs,
                                        uint32_t sample_base, uint32_t* __restrict__ row_base, uint32_t* __restrict__ row_sample) {
  const uint32_t p = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= n_inputs) return;
  const uint32_t base = (uint32_t)(local_excl[p] + block_excl[p / scan_block]), cnt = row_count[p];
  if (lane == 0) row_base[p] = base;
  for (uint32_t r = lane; r < cnt; r += 32) row_sample[base + r] = p + sample_base;
}

}  // namespace b2t
