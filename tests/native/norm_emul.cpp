// norm_emul.cpp -- TEST ONLY: runs the device code of tokenizers_b200/csrc/norm_kernels.cuh on the host, one "thread"
// after the other, with the tables tokenizers_b200/csrc/host_tables.cu builds (compiled unchanged as C++ next to this file),
// so that the survivor refusal of N1 (norm_load_chunk -> norm_survivor_refused) and N3's offset mapping can be checked
// against the reference's per-character alignment without a GPU.  The CUDA keywords and intrinsics the header uses are
// shimmed below; the header itself is compiled unchanged.
//   g++ -O2 -std=c++17 -I/usr/local/cuda/include -Wno-attributes -shared -fPIC -include cuda_runtime.h -o libnorm_emul.so \
//       norm_emul.cpp -x c++ ../../tokenizers_b200/csrc/host_tables.cu
#include <stdint.h>
#include <string.h>
#include <cuda_runtime.h>

struct Dim3e { unsigned x = 0, y = 0, z = 0; };
static Dim3e blockIdx, threadIdx, blockDim;
#define __syncthreads() ((void)0)
#define __launch_bounds__(...)
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline unsigned atomicOr(unsigned* p, unsigned v) { unsigned o = *p; *p |= v; return o; }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) { s &= 31u; return s ? (lo >> s) | (hi << (32u - s)) : lo; }
static inline int __shfl_up_sync(unsigned, int v, unsigned) { return v; }   // (only the block scans use it; not called here)
#undef __shared__
#define __shared__ static

#include "../../tokenizers_b200/csrc/norm_kernels.cuh"
#include "../../tokenizers_b200/csrc/host_tables.h"

using namespace b2t;

static NormHost g_norm;
static NormTables g_t;

// Builds the table for the BertNormalizer flags (bits: 1 clean_text, 2 handle_chinese_chars, 4 strip_accents, 8 lowercase)
// the way the engine does.  Returns 0, or -1 when an image does not fit the kernels' bound.
extern "C" int b2t_emul_norm_tables(int flags) {
  g_norm = NormHost();
  build_bert_norm(flags & 1, flags & 2, flags & 4, flags & 8, &g_norm);
  g_t.blk = g_norm.blk.data(); g_t.ent = g_norm.ent.data(); g_t.pool = g_norm.pool.data(); g_t.ascii = g_norm.ascii.data();
  return g_norm.ok ? 0 : -1;
}

// N1's refusal for each of n_batches packed batches (batch b = bytes[batch_off[b], batch_off[b + 1])): every 8-byte thread
// chunk of the batch through norm_load_chunk, refused[b] = 1 if any raised ERR_NORM_UNSUPPORTED.  Also the image size and
// the character count N1 computes, summed per batch.
extern "C" void b2t_emul_norm_refused(const uint8_t* bytes, const uint64_t* batch_off, uint32_t n_batches, uint8_t* refused,
                                      uint64_t* n_out, uint64_t* n_chars) {
  for (uint32_t b = 0; b < n_batches; ++b) {
    const uint8_t* p = bytes + batch_off[b];
    const int64_t n = (int64_t)(batch_off[b + 1] - batch_off[b]);
    uint32_t err = 0u;
    uint64_t o = 0, c = 0;
    for (int64_t base = 0; base < n; base += NORM_PER_THREAD) {
      NormChunk ch;
      norm_load_chunk(p, n, base, g_t, g_t.ascii, ch, &err);
      o += (uint64_t)ch.n_out; c += (uint64_t)ch.n_chars;
    }
    refused[b] = (err & ERR_NORM_UNSUPPORTED) ? 1 : 0;
    n_out[b] = o; n_chars[b] = c;
  }
}

// N3 over n_docs documents, one warp per document and its 32 lanes one after the other: offsets (uint2 per token) are
// rewritten in place from byte offsets in the normalized document to character offsets in the original one.
extern "C" void b2t_emul_norm_offsets(const uint64_t* row_ptr, uint32_t n_docs, const uint64_t* doc_off_norm, const uint32_t* doc_char0,
                                      const uint32_t* src_char, uint32_t* offsets) {
  blockDim.x = 32;
  for (uint32_t d = 0; d < n_docs; ++d)
    for (unsigned lane = 0; lane < 32; ++lane) {
      blockIdx.x = d; threadIdx.x = lane;
      norm_offsets_kernel(row_ptr, n_docs, 0ull, doc_off_norm, doc_char0, src_char, reinterpret_cast<uint2*>(offsets));
    }
}
