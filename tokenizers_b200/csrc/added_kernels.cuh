// added_kernels.cuh -- added / special token extraction on the device, in front of the pre-tokenization scan.
//
// Replaces, for pipelines without a normalizer (paths relative to tokenizers/src of huggingface/tokenizers):
//   tokenizer/added_vocabulary.rs:523-564  extract_and_normalize: the text is split on the added tokens with
//                                          normalized == false first, then every remaining piece on the normalized ones
//   tokenizer/added_vocabulary.rs:430-490  find_matches: leftmost-longest, non-overlapping matches (the reference builds an
//                                          Aho-Corasick automaton), filtered by single_word, widened by lstrip / rstrip
//   tokenizer/added_vocabulary.rs:99-125   the \w / \s tests of those rules (Rust regex classes)
//
// The reference cuts the sequence into pieces, pre-tokenizes every plain piece on its own and gives an added token's
// span its id directly.  Here nothing is cut or re-packed: three bitmaps tell the kernels that follow what happened.
//   hard_bits   document starts + starts and ends of added-token spans: the pre-tokenization scan treats them all as
//               "a new string starts here" (its regex never sees across them)
//   inner_bits  bytes of a span after its first: the scan clears every split there, the span is ONE pre-token
//   added_bits  first byte of a span: the page kernel takes the token id from the page's list (added_head / added_pool:
//               one linked list per 2 KB page, entries bump-allocated) instead of running the model
// A1 (added_scan) marks the positions whose first two bytes start some added token -- a filter, 1 B read per input byte;
// A2 (added_resolve), one thread per document that holds a candidate, walks them in order exactly like find_matches.
// What does not fit (a span over 256 bytes, more spans than one per 16 input bytes, the reference's overlapping-span corner
// after an rstrip) raises ERR_ADDED_UNSUPPORTED: the call fails with B2T_ERR_UNSUPPORTED, nothing is approximated.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "pretok_logic.cuh"

namespace b2t {

constexpr int ADDED_MAX_SPAN = 256;       // bytes (after lstrip / rstrip); the page kernel's halo
enum { ERR_ADDED_UNSUPPORTED = 8u };
constexpr uint32_t ADDED_NIL = 0xFFFFFFFFu;
enum { ADDED_SINGLE_WORD = 1u, ADDED_LSTRIP = 2u, ADDED_RSTRIP = 4u };

struct AddedTables {
  // tokens of set 0 (normalized == false) then set 1 (normalized == true), each set sorted by length, longest first
  const uint8_t* tok_bytes; const uint32_t* tok_off; const uint32_t* tok_id; const uint8_t* tok_flags;
  uint32_t set_begin[3];        // tokens of set s: [set_begin[s], set_begin[s + 1])
  const uint32_t* first_bits;   // [2][8]     bit b: some token of the set starts with byte b
  const uint32_t* pair_bits;    // [2][2048]  bit (b0 | b1 << 8): some token of the set starts with b0 b1 (one-byte tokens: every b1)
  const uint32_t* cls_rust;     // class table of the Rust regex crate (\w = CLS_L, \s = CLS_S), 2 bits per code point
  uint32_t n_first;             // distinct first bytes over both sets if there are at most 4 of them (else 0): ...
  uint32_t first_bcast[4];      // ... each repeated in the four bytes of a word, for a SWAR test of whole chunks
};

// ------------------------------------------------------------------------------------------------ A1: candidates
__device__ __forceinline__ void added_scan_chunk(const uint8_t* __restrict__ bytes, int64_t n, const AddedTables& T, const uint32_t* s_first,
                                                 int64_t c, int64_t base, uint32_t& m0, uint32_t& m1);

// cand_any: one bit per 32-byte chunk (bit c of the bitmap: cand0[c] | cand1[c] != 0), so that A2 can dismiss a document
// that holds no candidate with one or two loads.
__global__ void __launch_bounds__(256) added_scan_kernel(const uint8_t* __restrict__ bytes, int64_t n, const AddedTables T,
                                                         uint32_t* __restrict__ cand0, uint32_t* __restrict__ cand1, uint32_t* __restrict__ cand_any) {
  __shared__ uint32_t s_first[16];
  if (threadIdx.x < 16) s_first[threadIdx.x] = T.first_bits[threadIdx.x];
  __syncthreads();
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t base = c * CHUNK;
  uint32_t m0 = 0u, m1 = 0u;
  if (base < n) added_scan_chunk(bytes, n, T, s_first, c, base, m0, m1);
  if (base < n) { cand0[c] = m0; cand1[c] = m1; }
  const uint32_t any = __ballot_sync(0xFFFFFFFFu, (m0 | m1) != 0u);
  if ((threadIdx.x & 31) == 0 && base < n) cand_any[c >> 5] = any;   // (lane 0 holds the warp's first chunk)
}

__device__ __forceinline__ void added_scan_chunk(const uint8_t* __restrict__ bytes, int64_t n, const AddedTables& T, const uint32_t* s_first,
                                                 int64_t c, int64_t base, uint32_t& m0, uint32_t& m1) {
  uint32_t w[9];
  if (base + CHUNK + 4 <= n) {
    const uint4* q = reinterpret_cast<const uint4*>(bytes + base);
    const uint4 a = __ldg(q), b = __ldg(q + 1);
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
    w[8] = __ldg(reinterpret_cast<const uint32_t*>(bytes + base + CHUNK));
  } else {
#pragma unroll
    for (int j = 0; j < 9; ++j) {
      uint32_t v = 0;
      for (int k = 0; k < 4; ++k) { const int64_t p = base + 4 * j + k; if (p < n) v |= (uint32_t)__ldg(bytes + p) << (8 * k); }
      w[j] = v;
    }
  }
  if (T.n_first) {
    // special tokens start with a handful of bytes ('<', '['): a chunk that holds none of them has no candidate
    uint32_t any = 0u;
    for (uint32_t f = 0; f < T.n_first; ++f) {
      const uint32_t bc = T.first_bcast[f];
#pragma unroll
      for (int j = 0; j < 8; ++j) { const uint32_t x = w[j] ^ bc; any |= (x - 0x01010101u) & ~x & 0x80808080u; }   // a zero byte of x
    }
    if (!any) return;
  }
  const bool has1 = T.set_begin[2] > T.set_begin[1];
#pragma unroll
  for (int i = 0; i < CHUNK; ++i) {
    const uint32_t two = __funnelshift_r(w[i >> 2], w[(i >> 2) + 1], 8 * (i & 3)) & 0xFFFFu;   // bytes i, i + 1 (0 past the end)
    const uint32_t b0 = two & 0xFFu;
    if ((s_first[b0 >> 5] >> (b0 & 31)) & 1u) { if ((__ldg(T.pair_bits + (two >> 5)) >> (two & 31)) & 1u) m0 |= 1u << i; }
    if (has1 && ((s_first[8 + (b0 >> 5)] >> (b0 & 31)) & 1u)) { if ((__ldg(T.pair_bits + 2048 + (two >> 5)) >> (two & 31)) & 1u) m1 |= 1u << i; }
  }
  const int64_t lim = n - base;
  if (lim < CHUNK) { const uint32_t valid = (1u << (int)lim) - 1u; m0 &= valid; m1 &= valid; }
}

// ------------------------------------------------------------------------------------------------ A2: resolution
struct AddedOut {
  uint32_t* hard_bits; uint32_t* inner_bits; uint32_t* added_bits;
  uint32_t* head;         // [n_pages]: index of the page's first list entry, ADDED_NIL = none
  uint2* pool;            // entries {(start & (PAGE - 1)) | id << 11, next}
  uint32_t* pool_used; uint32_t pool_cap;
  uint32_t* err;
};

struct AddedCtx {
  const uint8_t* bytes; const AddedTables* T; const uint32_t* cand[2]; AddedOut o;
  int64_t doc_end;
};

__device__ __forceinline__ void set_bit(uint32_t* bits, int64_t p) { atomicOr(bits + (p >> 5), 1u << (p & 31)); }

// smallest position in [pos, limit) whose bit is set, or limit
__device__ __forceinline__ int64_t next_bit(const uint32_t* __restrict__ bits, int64_t pos, int64_t limit) {
  if (pos >= limit) return limit;
  int64_t wi = pos >> 5;
  uint32_t v = __ldg(bits + wi) & ~bits_below((int)(pos & 31));
  const int64_t wl = (limit - 1) >> 5;
  while (true) {
    if (v) { const int64_t p = wi * 32 + (__ffs((int)v) - 1); return p < limit ? p : limit; }
    if (++wi > wl) return limit;
    v = __ldg(bits + wi);
  }
}

// (code point, length) of the character that starts at p (p < limit, valid UTF-8)
__device__ __forceinline__ uint32_t char_at(const uint8_t* __restrict__ b, int64_t p, int64_t limit, int* len) {
  const uint32_t b0 = b[p];
  if (b0 < 0x80u) { *len = 1; return b0; }
  const int n = b0 < 0xE0u ? 2 : (b0 < 0xF0u ? 3 : 4);
  uint32_t cp = b0 & (0x7Fu >> n);
  for (int k = 1; k < n; ++k) cp = (cp << 6) | (p + k < limit ? (b[p + k] & 0x3Fu) : 0u);
  *len = n;
  return cp < 0x110000u ? cp : 0x10FFFFu;
}
// start of the character that ends at `end` (end > lo)
__device__ __forceinline__ int64_t char_start_before(const uint8_t* __restrict__ b, int64_t end, int64_t lo) {
  int64_t s = end - 1;
  while (s > lo && (b[s] & 0xC0u) == 0x80u && end - s < 4) --s;
  return s;
}

// longest token of the set that matches at p and ends at or before limit; -1 if none
__device__ __forceinline__ int match_at(const uint8_t* __restrict__ b, const AddedTables& T, int set, int64_t p, int64_t limit) {
  for (uint32_t t = T.set_begin[set]; t < T.set_begin[set + 1]; ++t) {
    const uint32_t o = T.tok_off[t], len = T.tok_off[t + 1] - o;
    if ((int64_t)len > limit - p) continue;
    bool same = true;
    for (uint32_t i = 0; i < len; ++i) if (T.tok_bytes[o + i] != b[p + i]) { same = false; break; }
    if (same) return (int)t;
  }
  return -1;
}

__device__ __forceinline__ void emit_span(const AddedCtx& c, int64_t start, int64_t stop, uint32_t id) {
  if (stop - start > ADDED_MAX_SPAN) { atomicOr(c.o.err, ERR_ADDED_UNSUPPORTED); return; }
  const int64_t page = start / PAGE;
  const uint32_t k = atomicAdd(c.o.pool_used, 1u);
  if (k >= c.o.pool_cap) { atomicOr(c.o.err, ERR_ADDED_UNSUPPORTED); return; }
  c.o.pool[k] = make_uint2((uint32_t)(start & (PAGE - 1)) | (id << 11), atomicExch(c.o.head + page, k));
  set_bit(c.o.added_bits, start);
  set_bit(c.o.hard_bits, start);
  if (stop < c.doc_end) set_bit(c.o.hard_bits, stop);
  for (int64_t p = start + 1; p < stop; ++p) set_bit(c.o.inner_bits, p);
}

// find_matches (added_vocabulary.rs:430-490) on the sentence [pa, pb) with token set `set`.  Plain pieces between the
// matches of set 0 are searched for set 1 (extract_and_normalize's second pass); plain pieces of set 1 need no action.
__device__ void added_find(const AddedCtx& c, int set, int64_t pa, int64_t pb) {
  const uint8_t* __restrict__ b = c.bytes;
  const AddedTables& T = *c.T;
  const bool has_set = T.set_begin[set + 1] > T.set_begin[set];
  int64_t start_offset = pa, scan = pa;
  while (has_set) {
    const int64_t p = next_bit(c.cand[set], scan, pb);
    if (p >= pb) break;
    const int t = match_at(b, T, set, p, pb);
    if (t < 0) { scan = p + 1; continue; }
    int64_t start = p, stop = p + (int64_t)(T.tok_off[t + 1] - T.tok_off[t]);
    scan = stop;   // the automaton goes on behind the match, whatever happens to it below
    const uint32_t fl = T.tok_flags[t];
    if (fl & ADDED_SINGLE_WORD) {
      bool start_space = start == pa, stop_space = stop == pb;
      int len;
      if (!start_space) start_space = class_of(T.cls_rust, char_at(b, char_start_before(b, start, pa), pb, &len)) != CLS_L;
      if (!stop_space) stop_space = class_of(T.cls_rust, char_at(b, stop, pb, &len)) != CLS_L;
      if (!start_space || !stop_space) continue;
    }
    if (fl & ADDED_LSTRIP) {
      int64_t e = start;
      while (e > pa) {
        int len;
        const int64_t s = char_start_before(b, e, pa);
        if (class_of(T.cls_rust, char_at(b, s, pb, &len)) != CLS_S) break;
        e = s;
      }
      start = e > start_offset ? e : start_offset;
    }
    if (fl & ADDED_RSTRIP) {
      while (stop < pb) {
        int len;
        if (class_of(T.cls_rust, char_at(b, stop, pb, &len)) != CLS_S) break;
        stop += len;
      }
    }
    if (start < start_offset) { atomicOr(c.o.err, ERR_ADDED_UNSUPPORTED); return; }   // the reference emits overlapping splits here
    if (set == 0 && start_offset < start) added_find(c, 1, start_offset, start);
    emit_span(c, start, stop, T.tok_id[t]);
    start_offset = stop;
  }
  if (set == 0 && start_offset < pb) added_find(c, 1, start_offset, pb);
}

__global__ void __launch_bounds__(128) added_resolve_kernel(const uint8_t* __restrict__ bytes, const uint64_t* __restrict__ doc_off, uint32_t n_docs,
                                                            const AddedTables T, const uint32_t* __restrict__ cand0, const uint32_t* __restrict__ cand1,
                                                            const uint32_t* __restrict__ cand_any, AddedOut o) {
  const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n_docs) return;
  const int64_t a = (int64_t)doc_off[d], b = (int64_t)doc_off[d + 1];
  if (a >= b) return;
  if (next_bit(cand_any, a / CHUNK, (b - 1) / CHUNK + 1) >= (b - 1) / CHUNK + 1) return;   // nearly every document: no chunk of it holds a candidate
  AddedCtx c;
  c.bytes = bytes; c.T = &T; c.cand[0] = cand0; c.cand[1] = cand1; c.o = o; c.doc_end = b;
  added_find(c, 0, a, b);
}

}  // namespace b2t
