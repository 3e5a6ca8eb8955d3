// overflow_emul.cpp -- TEST ONLY: compiles the device code of tokenizers_b200/csrc/dense_kernels.cuh for the host and runs
// the overflow path of dense mode as the engine launches it -- dense_count_kernel, an exclusive scan of the row counts,
// dense_row_sample_kernel, then the OVER (+ OFFS) instantiation of dense_rows_kernel / dense_pair_rows_kernel -- one
// thread at a time, plus the part algebra on its own (seq_parts, seq_part, pair_row_part).  The tests check it against the
// shim's host restatement of the reference (truncation_spans, pairs.post_process) without a GPU.  The CUDA keywords and
// intrinsics the header uses are shimmed below; the header itself is compiled unchanged.
//   g++ -O2 -std=c++17 -I/usr/local/cuda/include -Wno-attributes -shared -fPIC -o liboverflow_emul.so overflow_emul.cpp
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

// runs f for every thread of a grid of `threads` threads in blocks of `block`, one thread after the other.  The warp
// kernels need nothing from their lanes' order; the count pass runs in blocks of one thread, so that its warp maximum
// (a shuffle that returns the thread's own value here) is every thread's own.
template <class F>
static void launch(uint64_t threads, unsigned block, F&& f) {
  blockDim.x = block;
  for (uint64_t t = 0; t < threads; ++t) {
    blockIdx.x = (unsigned)(t / block); threadIdx.x = (unsigned)(t % block);
    f();
  }
}

extern "C" uint32_t b2t_emul_seq_parts(uint32_t n, uint32_t m, uint32_t s) { return seq_parts(n, m, s); }
extern "C" void b2t_emul_seq_part(uint32_t n, uint32_t m, uint32_t s, int left, uint32_t k, uint32_t* first, uint32_t* len) {
  seq_part(n, m, s, left != 0, k, first, len);
}
extern "C" void b2t_emul_pair_row_part(uint32_t r, uint32_t ox, uint32_t oy, uint32_t* i, uint32_t* j) { pair_row_part(r, ox, oy, i, j); }

// The count pass: row_count[n_inputs] -> returns R; *max_all, *err (ERR_* bits), *stride_m as in the ctl block
extern "C" uint64_t b2t_emul_overflow_count(const uint64_t* row_ptr, uint32_t n_inputs, uint32_t pairs, uint32_t budget, uint32_t strategy,
                                            uint32_t stride, uint32_t n_special, uint32_t* row_count, uint32_t* max_all, uint32_t* err,
                                            uint32_t* stride_m) {
  *max_all = 0; *err = 0; *stride_m = 0;
  launch(n_inputs, 1, [&] { dense_count_kernel(row_ptr, n_inputs, pairs, budget, strategy, stride, n_special, row_count, max_all, err, stride_m); });
  uint64_t R = 0;
  for (uint32_t p = 0; p < n_inputs; ++p) R += row_count[p];
  return R;
}

// The rows: R rows of width L from the count pass's row_count.  Pairs: special[] = pre, mid, post back to back (id | type
// << 24), b_first / type_x / type_y as PairDenseSpec; single sequences: special[] = pre, post (ids), type ids not written.
// offsets = NULL: no offset rows.
extern "C" void b2t_emul_overflow_rows(const uint32_t* ids, const uint32_t* offsets, const uint64_t* row_ptr, uint32_t n_inputs, uint32_t pairs,
                                       const uint32_t* row_count, uint32_t R, uint32_t L, uint32_t budget, uint32_t strategy, uint32_t stride,
                                       int trunc_left, int pad_left, uint32_t pad_id, uint32_t pad_type, uint32_t n_pre, uint32_t n_mid,
                                       uint32_t n_post, const uint32_t* special, uint32_t b_first, uint32_t type_x, uint32_t type_y,
                                       uint32_t type_oa, uint32_t type_ob, uint32_t sample_base, uint32_t* out_ids, uint8_t* out_type,
                                       uint8_t* out_mask, uint32_t* out_len, uint32_t* out_sample, uint32_t* out_off) {
  // the two-level scan of the engine, as one level: local_excl = the exclusive prefix, block_excl = 0
  std::vector<unsigned long long> lexcl(n_inputs + 1, 0ull), bexcl(n_inputs / 1024 + 2, 0ull);
  for (uint32_t p = 0; p < n_inputs; ++p) lexcl[p + 1] = lexcl[p] + row_count[p];
  std::vector<uint32_t> row_base(n_inputs + 1);
  launch((uint64_t)n_inputs * 32, 256, [&] {
    dense_row_sample_kernel(row_count, lexcl.data(), bexcl.data(), 1024, n_inputs, sample_base, row_base.data(), out_sample);
  });
  DenseOverflow O{out_sample, row_base.data(), sample_base, stride, b_first ? type_ob : type_oa, b_first ? type_oa : type_ob,
                  reinterpret_cast<const uint2*>(offsets), reinterpret_cast<uint2*>(out_off)};
  if (pairs) {
    PairDenseSpec S;
    memset(&S, 0, sizeof(S));
    S.L = L; S.budget = budget; S.strategy = strategy; S.pad_id = pad_id; S.pad_type = pad_type; S.trunc_left = trunc_left; S.pad_left = pad_left;
    S.b_first = b_first; S.type_x = type_x; S.type_y = type_y; S.n_pre = n_pre; S.n_mid = n_mid; S.n_post = n_post;
    memcpy(S.special, special, (n_pre + n_mid + n_post) * 4);
    launch((uint64_t)R * 32, 256, [&] {
      if (offsets) dense_pair_rows_kernel<true, true>(ids, row_ptr, R, S, out_ids, out_type, out_mask, out_len, O);
      else dense_pair_rows_kernel<true, false>(ids, row_ptr, R, S, out_ids, out_type, out_mask, out_len, O);
    });
  } else {
    DenseSpec S;
    memset(&S, 0, sizeof(S));
    S.L = L; S.keep_max = budget; S.pad_id = pad_id; S.n_pre = n_pre; S.n_post = n_post; S.trunc_left = trunc_left; S.pad_left = pad_left;
    memcpy(S.pre, special, n_pre * 4); memcpy(S.post, special + n_pre, n_post * 4);
    launch((uint64_t)R * 32, 256, [&] {
      if (offsets) dense_rows_kernel<true, true>(ids, row_ptr, R, S, out_ids, out_mask, out_len, nullptr, O);
      else dense_rows_kernel<true, false>(ids, row_ptr, R, S, out_ids, out_mask, out_len, nullptr, O);
    });
  }
}
