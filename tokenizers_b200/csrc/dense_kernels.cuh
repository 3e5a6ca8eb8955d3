// dense_kernels.cuh -- the post-path steps of a single-sequence batch on the device: special-token template, truncation
// and padding, emitted as dense [n_docs, L] id / attention-mask tensors straight from the token CSR.
//
// Replaces, for batches of single sequences (paths relative to tokenizers/src of huggingface/tokenizers):
//   tokenizer/mod.rs:1265-1317       TokenizerImpl::post_process: truncate to max_length - n_added_tokens, template, padding
//   utils/truncation.rs:70-166       truncate_encodings, single sequence: keep the first (direction right) or the last
//                                    (direction left) max_length tokens -- the kept part of Encoding::truncate
//                                    (tokenizer/encoding.rs:307-388); overflowing parts are not part of a dense batch
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

// One warp per row.  row_ptr is the (chunk-relative) CSR of `ids`; rows are written at out_* + d * L.
// A row that does not fit L (padding to a fixed length without truncation) raises bit 0 of *err and is cut -- the host
// turns that into an error, the reference would return a longer row there.
__global__ void dense_rows_kernel(const uint32_t* __restrict__ ids, const uint64_t* __restrict__ row_ptr, uint32_t n_docs, const DenseSpec S,
                                  uint32_t* __restrict__ out_ids, uint8_t* __restrict__ out_mask, uint32_t* __restrict__ out_len,
                                  uint32_t* __restrict__ err) {
  const uint32_t d = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (d >= n_docs) return;
  const uint64_t a = row_ptr[d], cnt = row_ptr[d + 1] - a;
  uint32_t keep = (uint32_t)(cnt < (uint64_t)S.keep_max ? cnt : (uint64_t)S.keep_max);
  uint32_t len = S.n_pre + keep + S.n_post;
  if (len > S.L) {
    if (lane == 0 && err) atomicOr(err, 1u);
    keep = S.L > S.n_pre + S.n_post ? S.L - S.n_pre - S.n_post : 0u;
    len = S.n_pre + keep + S.n_post;
    if (len > S.L) return;
  }
  const uint64_t src = a + (S.trunc_left ? cnt - keep : 0ull);
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
    row[j] = v;
    if (mrow) mrow[j] = k < len ? 1 : 0;
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
__global__ void dense_pair_rows_kernel(const uint32_t* __restrict__ ids, const uint64_t* __restrict__ row_ptr, uint32_t n_pairs,
                                       const __grid_constant__ PairDenseSpec S, uint32_t* __restrict__ out_ids, uint8_t* __restrict__ out_type,
                                       uint8_t* __restrict__ out_mask, uint32_t* __restrict__ out_len) {
  const uint32_t p = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= n_pairs) return;
  const uint64_t a = row_ptr[2 * p], b = row_ptr[2 * p + 1], c = row_ptr[2 * p + 2];
  const uint32_t n1 = (uint32_t)(b - a), n2 = (uint32_t)(c - b);
  uint32_t k1, k2;
  pair_keep(n1, n2, S.budget, S.strategy, &k1, &k2);   // (a SequenceTooShort pair fails the batch: its row does not matter)
  const uint64_t src1 = a + (S.trunc_left ? n1 - k1 : 0u), src2 = b + (S.trunc_left ? n2 - k2 : 0u);
  const uint64_t src_x = S.b_first ? src2 : src1, src_y = S.b_first ? src1 : src2;
  const uint32_t kx = S.b_first ? k2 : k1, ky = S.b_first ? k1 : k2;
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
    if (k < e0 || (k >= e1 && k < e2) || (k >= e3 && k < len)) {
      const uint32_t s = S.special[k < e0 ? k : (k < e2 ? e0 + (k - e1) : e0 + S.n_mid + (k - e3))];
      v = s & 0xFFFFFFu; t = s >> 24;
    } else if (k < e1) {
      v = ids[src_x + (k - e0)]; t = S.type_x;
    } else if (k < e3) {
      v = ids[src_y + (k - e2)]; t = S.type_y;
    }
    row[j] = v;
    trow[j] = (uint8_t)t;
    if (mrow) mrow[j] = k < len ? 1 : 0;
  }
  if (lane == 0) out_len[p] = len;
}

}  // namespace b2t
