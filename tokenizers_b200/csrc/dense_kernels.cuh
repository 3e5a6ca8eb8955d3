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

}  // namespace b2t
