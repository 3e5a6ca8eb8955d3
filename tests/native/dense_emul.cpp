// dense_emul.cpp -- TEST ONLY: compiles the device code of tokenizers_b200/csrc/dense_kernels.cuh for the host and exports
// the pair truncation algebra (pair_keep) the pair kernels run, so that it can be checked exhaustively against the plain
// restatement of the reference (tests/pair_oracle.py) without a GPU.  The CUDA keywords and intrinsics the header uses
// are shimmed below; the header itself is compiled unchanged.
//   g++ -O2 -std=c++17 -I/usr/local/cuda/include -Wno-attributes -shared -fPIC -o libdense_emul.so dense_emul.cpp
#include <stdint.h>
#include <cuda_runtime.h>

struct Dim3e { unsigned x = 0, y = 0, z = 0; };
static Dim3e blockIdx, threadIdx, blockDim;
static inline unsigned atomicOr(unsigned* p, unsigned v) { unsigned o = *p; *p |= v; return o; }
static inline unsigned atomicMax(unsigned* p, unsigned v) { unsigned o = *p; if (v > o) *p = v; return o; }
static inline unsigned __shfl_xor_sync(unsigned, unsigned v, int) { return v; }   // (only the kernels use it; not called here)
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }

#include "../../tokenizers_b200/csrc/dense_kernels.cuh"

using namespace b2t;

// pair_keep over n inputs: strategy PAIR_* (0 longest_first, 1 only_first, 2 only_second), budget 0xFFFFFFFF = no truncation;
// ok[i] = 0 where the batch would fail with SequenceTooShort
extern "C" void b2t_emul_pair_keep(uint32_t n, const uint32_t* n1, const uint32_t* n2, const uint32_t* budget, const uint32_t* strategy,
                                   uint32_t* k1, uint32_t* k2, uint8_t* ok) {
  for (uint32_t i = 0; i < n; ++i) ok[i] = pair_keep(n1[i], n2[i], budget[i], strategy[i], &k1[i], &k2[i]) ? 1 : 0;
}
