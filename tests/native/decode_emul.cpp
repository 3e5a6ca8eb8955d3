// decode_emul.cpp -- TEST ONLY: runs the lossy UTF-8 classifier of tokenizers_b200/csrc/decode_kernels.cuh (compiled unchanged
// as host code) the way D2 counts and D3 rewrites a row, so that it can be checked against Python's
// bytes.decode("utf-8", "replace") without a GPU.
//   g++ -O2 -std=c++17 -I/usr/local/cuda/include -shared -fPIC -o libdecode_emul.so decode_emul.cpp
#include <stdint.h>
#include <vector_types.h>

#include "../../tokenizers_b200/csrc/decode_kernels.cuh"

using namespace b2t;

// Rows of in (row r = in[off[r] .. off[r+1])) through the lossy rule, each on its own, into out (capacity 3 x in) at
// out_off.  Returns the bytes written.
extern "C" uint64_t b2t_emul_lossy(const uint8_t* in, const uint64_t* off, uint32_t n_rows, uint8_t* out, uint64_t* out_off) {
  uint64_t pos = 0;
  for (uint32_t r = 0; r < n_rows; ++r) {
    out_off[r] = pos;
    const uint8_t* row = in + off[r];
    const int64_t len = (int64_t)(off[r + 1] - off[r]);
    uint64_t count = 0;   // D2's count of the row
    for (int64_t p = 0; p < len; ++p) count += lossy_bytes(lossy_class(row, p, len));
    for (int64_t p = 0; p < len; ++p) {   // D3's rewrite of the row
      const int c = lossy_class(row, p, len);
      if (c == LOSSY_VALID) out[pos++] = row[p];
      else if (c == LOSSY_REPLACE) { out[pos++] = 0xEF; out[pos++] = 0xBF; out[pos++] = 0xBD; }
    }
    if (pos - out_off[r] != count) return ~0ull;   // the count and the rewrite disagree
  }
  out_off[n_rows] = pos;
  return pos;
}
