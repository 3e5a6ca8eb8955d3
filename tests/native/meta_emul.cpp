// meta_emul.cpp -- TEST ONLY: compiles the device code of tokenizers_b200/csrc/dense_kernels.cuh for the host and runs
// the META instantiations of dense_rows_kernel / dense_pair_rows_kernel (row metadata: trimmed offset rows, special-tokens
// mask, sequence ids, word ids) as the engine launches them -- with overflowing parts behind dense_count_kernel and
// dense_row_sample_kernel, or on the kept parts alone -- one thread at a time, plus the trim rules on their own
// (trim_span, added_trim_counts).  The tests check it against the shim's host restatement of the reference (trim_spans,
// _span_spaces, pairs.post_process) without a GPU.  The CUDA keywords and intrinsics the header uses are shimmed below; the
// header itself is compiled unchanged.
//   g++ -O2 -std=c++17 -I/usr/local/cuda/include -Wno-attributes -shared -fPIC -o libmeta_emul.so meta_emul.cpp
#include <stdint.h>
#include <string.h>
#include <vector>
#include <cuda_runtime.h>

struct Dim3e { unsigned x = 0, y = 0, z = 0; };
static Dim3e blockIdx, threadIdx, blockDim;
static inline unsigned atomicOr(unsigned* p, unsigned v) { unsigned o = *p; *p |= v; return o; }
static inline unsigned atomicMax(unsigned* p, unsigned v) { unsigned o = *p; if (v > o) *p = v; return o; }
static inline unsigned __shfl_xor_sync(unsigned, unsigned v, int) { return v; }   // one thread per "warp": see launch()
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }

#include "../../tokenizers_b200/csrc/dense_kernels.cuh"

using namespace b2t;

// runs f for every thread of a grid of `threads` threads in blocks of `block`, one thread after the other (the count pass
// runs in blocks of one thread, so that its warp maximum -- a shuffle that returns the thread's own value here -- is every
// thread's own)
template <class F>
static void launch(uint64_t threads, unsigned block, F&& f) {
  blockDim.x = block;
  for (uint64_t t = 0; t < threads; ++t) {
    blockIdx.x = (unsigned)(t / block); threadIdx.x = (unsigned)(t % block);
    f();
  }
}

extern "C" void b2t_emul_trim_span(uint32_t o0, uint32_t o1, uint32_t ld, uint32_t tr, int first, int aps, uint32_t* out) {
  const uint2 o = trim_span(make_uint2(o0, o1), ld, tr, first != 0, aps != 0);
  out[0] = o.x; out[1] = o.y;
}

// 1 = counts in *ld / *tr, 0 = ambiguous
extern "C" int b2t_emul_added_trim_counts(uint32_t S, uint32_t chars, uint32_t lc, uint32_t tc, uint32_t flags, uint32_t* ld, uint32_t* tr) {
  const AddedTrim a{0u, chars, lc | tc << 16, flags};
  return added_trim_counts(S, a, ld, tr) ? 1 : 0;
}

// The count pass (as the engine runs it with overflowing parts): row_count[n_inputs] -> R; *max_all, *err
extern "C" uint64_t b2t_emul_meta_count(const uint64_t* row_ptr, uint32_t n_inputs, uint32_t pairs, uint32_t budget, uint32_t strategy,
                                        uint32_t stride, uint32_t n_special, uint32_t* row_count, uint32_t* max_all, uint32_t* err) {
  uint32_t stride_m = 0;
  *max_all = 0; *err = 0;
  launch(n_inputs, 1, [&] { dense_count_kernel(row_ptr, n_inputs, pairs, budget, strategy, stride, n_special, row_count, max_all, err, &stride_m); });
  uint64_t R = 0;
  for (uint32_t p = 0; p < n_inputs; ++p) R += row_count[p];
  return R;
}

// The META rows: over = 1: R rows from the count pass's row_count (the <1, *, 1> instantiations); over = 0: one row per
// input (<0, *, 1>).  Spec arguments as overflow_emul.cpp's b2t_emul_overflow_rows.  offsets = NULL: no offset rows;
// trim_vocab = NULL: no trimming, else trim_added = n_added entries (id, chars, lead | trail << 16, TRIM_* flags) by
// ascending id; word_ids = NULL: no word rows.  Null outputs are not written.  -> the error bits the kernels raised.
extern "C" uint32_t b2t_emul_meta_rows(const uint32_t* ids, const uint32_t* offsets, const uint32_t* word_ids, const uint64_t* row_ptr, uint32_t n_inputs,
                                       uint32_t pairs, uint32_t over, const uint32_t* row_count, uint32_t R, uint32_t L, uint32_t budget, uint32_t strategy,
                                       uint32_t stride, int trunc_left, int pad_left, uint32_t pad_id, uint32_t pad_type, uint32_t n_pre, uint32_t n_mid,
                                       uint32_t n_post, const uint32_t* special, uint32_t b_first, uint32_t type_x, uint32_t type_y, uint32_t type_oa,
                                       uint32_t type_ob, const uint32_t* trim_vocab, const uint32_t* trim_added, uint32_t n_added, uint32_t aps,
                                       uint32_t* out_ids, uint8_t* out_type, uint8_t* out_mask, uint32_t* out_len, uint32_t* out_sample,
                                       uint32_t* out_off, uint8_t* out_special, int8_t* out_seq, uint32_t* out_word) {
  std::vector<unsigned long long> lexcl(n_inputs + 1, 0ull), bexcl(n_inputs / 1024 + 2, 0ull);
  std::vector<uint32_t> row_base(n_inputs + 1);
  if (over) {   // the two-level scan of the engine, as one level: local_excl = the exclusive prefix, block_excl = 0
    for (uint32_t p = 0; p < n_inputs; ++p) lexcl[p + 1] = lexcl[p] + row_count[p];
    launch((uint64_t)n_inputs * 32, 256, [&] {
      dense_row_sample_kernel(row_count, lexcl.data(), bexcl.data(), 1024, n_inputs, 0u, row_base.data(), out_sample);
    });
  } else {
    R = n_inputs;
  }
  uint32_t err = 0;
  const DenseOverflow O{over ? out_sample : nullptr, over ? row_base.data() : nullptr, 0u, over ? stride : 0u, b_first ? type_ob : type_oa,
                        b_first ? type_oa : type_ob, reinterpret_cast<const uint2*>(offsets), reinterpret_cast<uint2*>(out_off)};
  const DenseMeta M{trim_vocab, reinterpret_cast<const AddedTrim*>(trim_added), n_added, aps, word_ids, out_special, out_seq,
                    word_ids ? out_word : nullptr, &err};
  const bool offs = offsets != nullptr;
  if (pairs) {
    PairDenseSpec S;
    memset(&S, 0, sizeof(S));
    S.L = L; S.budget = budget; S.strategy = strategy; S.pad_id = pad_id; S.pad_type = pad_type; S.trunc_left = trunc_left; S.pad_left = pad_left;
    S.b_first = b_first; S.type_x = type_x; S.type_y = type_y; S.n_pre = n_pre; S.n_mid = n_mid; S.n_post = n_post;
    memcpy(S.special, special, (n_pre + n_mid + n_post) * 4);
    launch((uint64_t)R * 32, 256, [&] {
      if (over && offs) dense_pair_rows_kernel<true, true, true>(ids, row_ptr, R, S, out_ids, out_type, out_mask, out_len, O, M);
      else if (over) dense_pair_rows_kernel<true, false, true>(ids, row_ptr, R, S, out_ids, out_type, out_mask, out_len, O, M);
      else if (offs) dense_pair_rows_kernel<false, true, true>(ids, row_ptr, R, S, out_ids, out_type, out_mask, out_len, O, M);
      else dense_pair_rows_kernel<false, false, true>(ids, row_ptr, R, S, out_ids, out_type, out_mask, out_len, O, M);
    });
  } else {
    DenseSpec S;
    memset(&S, 0, sizeof(S));
    S.L = L; S.keep_max = budget; S.pad_id = pad_id; S.n_pre = n_pre; S.n_post = n_post; S.trunc_left = trunc_left; S.pad_left = pad_left;
    memcpy(S.pre, special, n_pre * 4); memcpy(S.post, special + n_pre, n_post * 4);
    launch((uint64_t)R * 32, 256, [&] {
      if (over && offs) dense_rows_kernel<true, true, true>(ids, row_ptr, R, S, out_ids, out_mask, out_len, nullptr, O, M);
      else if (over) dense_rows_kernel<true, false, true>(ids, row_ptr, R, S, out_ids, out_mask, out_len, nullptr, O, M);
      else if (offs) dense_rows_kernel<false, true, true>(ids, row_ptr, R, S, out_ids, out_mask, out_len, nullptr, O, M);
      else dense_rows_kernel<false, false, true>(ids, row_ptr, R, S, out_ids, out_mask, out_len, nullptr, O, M);
    });
  }
  return err;
}
