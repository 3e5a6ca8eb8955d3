// dense_emul.cpp -- TEST ONLY: compiles the device code of tokenizers_b200/csrc/dense_kernels.cuh for the host and runs
// dense mode as the engine launches it, one thread at a time: the length pass (row_len_max_kernel / pair_len_max_kernel,
// or with overflowing parts dense_count_kernel and the scan of the row counts), dense_row_sample_kernel, and every
// <OVER, OFFS, META> instance of dense_rows_kernel / dense_pair_rows_kernel -- plus the algebra on its own (pair_keep,
// seq_parts, seq_part, pair_row_part, trim_span, added_trim_counts).  The tests check it against the plain restatements
// (tests/dense_oracle.py, oracle.dense_rows) without a GPU.  The CUDA keywords and intrinsics the header uses are shimmed
// below; the header itself is compiled unchanged.
//   g++ -O2 -std=c++17 -I/usr/local/cuda/include -Wno-attributes -shared -fPIC -o libdense_emul.so dense_emul.cpp
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
// kernels need nothing from their lanes' order; the length passes run in blocks of one thread, so that their warp maximum
// (a shuffle that returns the thread's own value here) is every thread's own.
template <class F>
static void launch(uint64_t threads, unsigned block, F&& f) {
  blockDim.x = block;
  for (uint64_t t = 0; t < threads; ++t) {
    blockIdx.x = (unsigned)(t / block); threadIdx.x = (unsigned)(t % block);
    f();
  }
}

// ------------------------------------------------------------------------------------------------------- algebra
// pair_keep over n inputs: strategy PAIR_* (0 longest_first, 1 only_first, 2 only_second), budget 0xFFFFFFFF = no truncation;
// ok[i] = 0 where the batch would fail with SequenceTooShort
extern "C" void b2t_emul_pair_keep(uint32_t n, const uint32_t* n1, const uint32_t* n2, const uint32_t* budget, const uint32_t* strategy,
                                   uint32_t* k1, uint32_t* k2, uint8_t* ok) {
  for (uint32_t i = 0; i < n; ++i) ok[i] = pair_keep(n1[i], n2[i], budget[i], strategy[i], &k1[i], &k2[i]) ? 1 : 0;
}

extern "C" uint32_t b2t_emul_seq_parts(uint32_t n, uint32_t m, uint32_t s) { return seq_parts(n, m, s); }
extern "C" void b2t_emul_seq_part(uint32_t n, uint32_t m, uint32_t s, int left, uint32_t k, uint32_t* first, uint32_t* len) {
  seq_part(n, m, s, left != 0, k, first, len);
}
extern "C" void b2t_emul_pair_row_part(uint32_t r, uint32_t ox, uint32_t oy, uint32_t* i, uint32_t* j) { pair_row_part(r, ox, oy, i, j); }

extern "C" void b2t_emul_trim_span(uint32_t o0, uint32_t o1, uint32_t ld, uint32_t tr, int first, int aps, uint32_t* out) {
  const uint2 o = trim_span(make_uint2(o0, o1), ld, tr, first != 0, aps != 0);
  out[0] = o.x; out[1] = o.y;
}

// 1 = counts in *ld / *tr, 0 = ambiguous
extern "C" int b2t_emul_added_trim_counts(uint32_t S, uint32_t chars, uint32_t lc, uint32_t tc, uint32_t flags, uint32_t* ld, uint32_t* tr) {
  const AddedTrim a{0u, chars, lc | tc << 16, flags};
  return added_trim_counts(S, a, ld, tr) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------- length pass
// As finish_tail runs it.  over = 0: row_len_max_kernel (budget = keep_max) or pair_len_max_kernel -> n_inputs rows,
// *max_len = the longest; over = 1: dense_count_kernel -> row_count[n_inputs] and R = their sum, *max_len = the longest
// of all rows, *stride_m.  *err: the ERR_* bits.
extern "C" uint64_t b2t_emul_dense_count(const uint64_t* row_ptr, uint32_t n_inputs, uint32_t pairs, uint32_t over, uint32_t budget,
                                         uint32_t strategy, uint32_t stride, uint32_t n_special, uint32_t* row_count, uint32_t* max_len,
                                         uint32_t* err, uint32_t* stride_m) {
  *max_len = 0; *err = 0; *stride_m = 0;
  if (!over) {
    launch(n_inputs, 1, [&] {
      if (pairs) pair_len_max_kernel(row_ptr, n_inputs, budget, strategy, n_special, max_len, err);
      else row_len_max_kernel(row_ptr, n_inputs, budget, n_special, max_len);
    });
    return n_inputs;
  }
  launch(n_inputs, 1, [&] { dense_count_kernel(row_ptr, n_inputs, pairs, budget, strategy, stride, n_special, row_count, max_len, err, stride_m); });
  uint64_t R = 0;
  for (uint32_t p = 0; p < n_inputs; ++p) R += row_count[p];
  return R;
}

// ---------------------------------------------------------------------------------------------------------- rows
struct Rows {
  const uint32_t* ids; const uint64_t* row_ptr;
  uint32_t pairs, R;
  PairDenseSpec P; DenseSpec S;
  uint32_t *out_ids; uint8_t *out_type, *out_mask; uint32_t* out_len;
  DenseOverflow O; DenseMeta M;
  uint32_t* err;
};

template <bool OVER, bool OFFS, bool META>
static void launch_rows(const Rows& a) {
  launch((uint64_t)a.R * 32, 256, [&] {
    if (a.pairs) dense_pair_rows_kernel<OVER, OFFS, META>(a.ids, a.row_ptr, a.R, a.P, a.out_ids, a.out_type, a.out_mask, a.out_len, a.O, a.M);
    else dense_rows_kernel<OVER, OFFS, META>(a.ids, a.row_ptr, a.R, a.S, a.out_ids, a.out_mask, a.out_len, a.err, a.O, a.M);
  });
}
using LaunchRows = void (*)(const Rows&);
constexpr LaunchRows LAUNCH_ROWS[2][2][2] = {   // [OVER][OFFS][META], as engine.cu
    {{launch_rows<false, false, false>, launch_rows<false, false, true>}, {launch_rows<false, true, false>, launch_rows<false, true, true>}},
    {{launch_rows<true, false, false>, launch_rows<true, false, true>}, {launch_rows<true, true, false>, launch_rows<true, true, true>}}};

// The rows of the instance <over, offs, meta>: R rows of width L, over = 1 from the count pass's row_count (the scan of the
// engine as one level, then dense_row_sample_kernel), else one per input.  The spec in the pair layout: special[] = pre,
// mid, post back to back, id | type << 24 for pairs; single sequences take budget as keep_max, pre / post ids from special[]
// (n_mid = 0) and write no type ids.  trim_vocab = NULL: no trimming, else trim_added = n_added entries (id, chars, lead |
// trail << 16, TRIM_* flags) by ascending id; word_ids = NULL: no word rows; null outputs are not written.  -> the error
// bits the row kernels raised (bit 0: a single-sequence row cut to L).
extern "C" uint32_t b2t_emul_dense_rows(const uint32_t* ids, const uint32_t* offsets, const uint32_t* word_ids, const uint64_t* row_ptr,
                                        uint32_t n_inputs, uint32_t pairs, uint32_t over, uint32_t offs, uint32_t meta, const uint32_t* row_count,
                                        uint32_t R, uint32_t L, uint32_t budget, uint32_t strategy, uint32_t stride, int trunc_left, int pad_left,
                                        uint32_t pad_id, uint32_t pad_type, uint32_t n_pre, uint32_t n_mid, uint32_t n_post, const uint32_t* special,
                                        uint32_t b_first, uint32_t type_x, uint32_t type_y, uint32_t type_oa, uint32_t type_ob,
                                        const uint32_t* trim_vocab, const uint32_t* trim_added, uint32_t n_added, uint32_t aps, uint32_t* out_ids,
                                        uint8_t* out_type, uint8_t* out_mask, uint32_t* out_len, uint32_t* out_sample, uint32_t* out_off,
                                        uint8_t* out_special, int8_t* out_seq, uint32_t* out_word) {
  std::vector<unsigned long long> lexcl(n_inputs + 1, 0ull), bexcl(n_inputs / 1024 + 2, 0ull);
  std::vector<uint32_t> row_base(n_inputs + 1);
  if (over) {   // the two-level scan of the engine, as one level: local_excl = the exclusive prefix, block_excl = 0
    for (uint32_t p = 0; p < n_inputs; ++p) lexcl[p + 1] = lexcl[p] + row_count[p];
    launch((uint64_t)n_inputs * 32, 256, [&] {
      dense_row_sample_kernel(row_count, lexcl.data(), bexcl.data(), 1024, n_inputs, 0u, row_base.data(), out_sample);
    });
  }
  uint32_t err = 0;
  Rows a;
  memset(&a, 0, sizeof(a));
  a.ids = ids; a.row_ptr = row_ptr; a.pairs = pairs; a.R = over ? R : n_inputs;
  a.out_ids = out_ids; a.out_type = out_type; a.out_mask = out_mask; a.out_len = out_len; a.err = &err;
  PairDenseSpec& P = a.P;
  P.L = L; P.budget = budget; P.strategy = strategy; P.pad_id = pad_id; P.pad_type = pad_type; P.trunc_left = trunc_left; P.pad_left = pad_left;
  P.b_first = b_first; P.type_x = type_x; P.type_y = type_y; P.n_pre = n_pre; P.n_mid = n_mid; P.n_post = n_post;
  memcpy(P.special, special, (n_pre + n_mid + n_post) * 4);
  DenseSpec& S = a.S;
  S.L = L; S.keep_max = budget; S.pad_id = pad_id; S.n_pre = n_pre; S.n_post = n_post; S.trunc_left = trunc_left; S.pad_left = pad_left;
  memcpy(S.pre, special, n_pre * 4); memcpy(S.post, special + n_pre, n_post * 4);
  if (over) {
    a.O.row_sample = out_sample; a.O.row_base = row_base.data(); a.O.stride = stride;
    a.O.type_ox = b_first ? type_ob : type_oa; a.O.type_oy = b_first ? type_oa : type_ob;
  }
  if (offs) { a.O.offsets = reinterpret_cast<const uint2*>(offsets); a.O.out_off = reinterpret_cast<uint2*>(out_off); }
  if (meta)
    a.M = DenseMeta{trim_vocab, reinterpret_cast<const AddedTrim*>(trim_added), n_added, aps, word_ids, out_special, out_seq,
                    word_ids ? out_word : nullptr, &err};
  LAUNCH_ROWS[over != 0][offs != 0][meta != 0](a);
  return err;
}
