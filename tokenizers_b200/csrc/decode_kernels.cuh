// decode_kernels.cuh -- D1-D3: token ids -> text (tokenizer/mod.rs:935-953 decode, per row of a batch).
//
// Every kept token's output depends only on its id and on whether it is the row's first kept token, so the host builds one
// table entry per id (host_tables.cu build_decoder_table, layout in b2t_tables.h DEC_*) and the kernels gather images:
//   D1 decode_count_kernel  one warp per row: the image bytes of the row (a ballot carried across the row's 32-token steps
//                           finds the first kept token); checks the row against the id buffer
//   (tile_scan_block_kernel / tile_scan_top_kernel over the row counts: each row's start in the text)
//   D2 decode_emit_kernel   one warp per row: gathers the images into shared memory step by step and stores them in whole
//                           16-byte blocks; for ByteLevel it then reads the row back, classifies it for from_utf8_lossy
//                           and counts its lossy length
//   D3 decode_lossy_kernel  only when D2 met an invalid byte: rewrites every row through the lossy rule (after a scan of
//                           D2's lossy counts)
//
// The lossy rule (String::from_utf8_lossy; equal to Python's bytes.decode("utf-8", "replace")): every maximal invalid
// subpart becomes U+FFFD.  It is local -- a byte's fate depends on at most 3 bytes on each side -- and never looks past
// the row's edges: each row is its own from_utf8_lossy.  The classifier below is plain host/device code, compiled for the
// host unchanged by tests/native/decode_emul.cpp.
#pragma once
#include <stdint.h>

#include "b2t_tables.h"

namespace b2t {

// ------------------------------------------------------------------------------------------------ lossy UTF-8 classifier
enum { LOSSY_VALID = 0, LOSSY_REPLACE = 1, LOSSY_SWALLOW = 2 };   // emit the byte / emit U+FFFD / emit nothing

// The sequence that starts at lead byte s[0] (avail bytes readable): *need = its length if it were complete; returns how
// many of its bytes form a valid prefix (0 for a byte that cannot start a sequence: 80-C1, F5-FF).  Unicode Table 3-7.
B2T_HDI int utf8_prefix(const uint8_t* s, int avail, int* need) {
  const uint32_t b = s[0];
  if (b < 0x80u) { *need = 1; return 1; }
  uint32_t lo = 0x80u, hi = 0xBFu;
  int n;
  if (b >= 0xC2u && b <= 0xDFu) n = 2;
  else if (b >= 0xE0u && b <= 0xEFu) { n = 3; if (b == 0xE0u) lo = 0xA0u; if (b == 0xEDu) hi = 0x9Fu; }
  else if (b >= 0xF0u && b <= 0xF4u) { n = 4; if (b == 0xF0u) lo = 0x90u; if (b == 0xF4u) hi = 0x8Fu; }
  else { *need = 1; return 0; }
  *need = n;
  int got = 1;
  for (; got < n && got < avail; ++got) {
    const uint32_t c = s[got];
    if (got == 1 ? (c < lo || c > hi) : (c & 0xC0u) != 0x80u) break;
  }
  return got;
}

// The fate of byte p of a row of len bytes under from_utf8_lossy: LOSSY_VALID (part of a valid character), LOSSY_REPLACE
// (first byte of a maximal invalid subpart) or LOSSY_SWALLOW (a later byte of one).  Reads row[p - 3 .. p + 3] at most,
// inside [0, len).  Only bytes outside 80-BF start a unit other than a lone byte, so the unit that holds a continuation
// byte starts at the nearest such byte behind it, at most 3 back.
B2T_HDI int lossy_class(const uint8_t* row, int64_t p, int64_t len) {
  const uint32_t b = row[p];
  if (b < 0x80u) return LOSSY_VALID;
  int64_t q = p;
  if ((b & 0xC0u) == 0x80u) {
    q = -1;
    for (int64_t k = p - 1; k >= 0 && k >= p - 3; --k)
      if ((row[k] & 0xC0u) != 0x80u) { q = k; break; }
    if (q < 0) return LOSSY_REPLACE;   // a lone continuation byte
  }
  int need;
  const int64_t avail = len - q < 4 ? len - q : 4;
  const int got = utf8_prefix(row + q, (int)avail, &need);
  if (got == need) return p - q < need ? LOSSY_VALID : LOSSY_REPLACE;
  const int unit = got > 0 ? got : 1;   // the maximal invalid subpart starting at q
  if (p - q >= unit) return LOSSY_REPLACE;
  return p == q ? LOSSY_REPLACE : LOSSY_SWALLOW;
}

// bytes a byte of that class turns into
B2T_HDI uint32_t lossy_bytes(int cls) { return cls == LOSSY_VALID ? 1u : cls == LOSSY_REPLACE ? 3u : 0u; }

#if defined(__CUDACC__)
// ------------------------------------------------------------------------------------------------ kernels
struct DecodeTable {
  const uint2* ent;      // DEC_* entries
  const uint8_t* pool;
  uint32_t n;            // entries: ids at or above are unknown
};
// Row r = ids[row_ptr[r] - id_base .. (row_len ? row_ptr[r] + row_len[r] : row_ptr[r + 1]) - id_base); ids holds
// [id_base, id_base + n_ids) of the caller's buffer
struct DecodeRows {
  const uint32_t* ids;
  const uint64_t* row_ptr;
  const uint32_t* row_len;
  uint64_t id_base, n_ids;
  uint32_t n_rows;
};
struct DecodeCtl {            // read back by the host
  unsigned long long total;   // image bytes of the batch (D1's scan)
  unsigned long long lossy;   // bytes after the lossy rewrite (ByteLevel, D3's scan)
  uint32_t err;               // DEC_ERR_*
  uint32_t bad;               // D2 met a byte that is not LOSSY_VALID
};
enum { DEC_ERR_ROWS = 1u, DEC_ERR_ROW_SIZE = 2u };
constexpr uint64_t DEC_MAX_ROW_TEXT = 1ull << 30;   // image bytes of one row (x3 after the lossy rewrite fits 32 bits)
constexpr int DEC_THREADS = 256, DEC_STAGE = 2048;   // per warp: shared staging of one step's images

__device__ __forceinline__ bool decode_row(const DecodeRows& R, uint32_t r, uint64_t* a, uint64_t* b) {
  const uint64_t s = R.row_ptr[r];
  const uint64_t e = R.row_len ? s + R.row_len[r] : R.row_ptr[r + 1];
  *a = s - R.id_base; *b = e - R.id_base;
  return s >= R.id_base && e >= s && e - R.id_base <= R.n_ids;
}

// One 32-token step of a row: the lane's token and its image (off, len) given whether a first kept token came before.
struct DecodeTok { uint32_t off, len; };
__device__ __forceinline__ DecodeTok decode_step(const DecodeTable& T, const DecodeRows& R, uint64_t i, uint64_t end, bool skip, bool* have_first) {
  const int lane = threadIdx.x & 31;
  uint2 e = make_uint2(0u, 0u);
  if (i < end) {
    const uint32_t id = __ldg(R.ids + i);
    if (id < T.n) e = __ldg(T.ent + id);
  }
  const bool kept = (e.y & DEC_EXISTS) && !(skip && (e.y & DEC_SKIP));
  const uint32_t ball = __ballot_sync(0xFFFFFFFFu, kept);
  const int first_lane = *have_first || !ball ? 32 : __ffs(ball) - 1;
  *have_first = *have_first || ball;
  const uint32_t l1 = e.y & DEC_LEN_MASK, l2 = (e.y >> DEC_LEN_BITS) & DEC_LEN_MASK;
  DecodeTok t;
  t.off = lane == first_lane ? e.x : e.x + l1;
  t.len = !kept ? 0u : lane == first_lane ? l1 : l2;
  return t;
}

__device__ __forceinline__ uint32_t warp_incl_sum(uint32_t v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int s = 1; s < 32; s <<= 1) { const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, v, s); if (lane >= s) v += o; }
  return v;
}

// D1: row r's image bytes -> count[r]; a row outside the id buffer or with row_ptr decreasing raises DEC_ERR_ROWS
__global__ void __launch_bounds__(DEC_THREADS) decode_count_kernel(const DecodeTable T, const DecodeRows R, uint32_t skip, uint32_t* __restrict__ count,
                                                                   DecodeCtl* __restrict__ ctl) {
  const uint32_t r = (uint32_t)(((uint64_t)blockIdx.x * DEC_THREADS + threadIdx.x) >> 5);
  if (r >= R.n_rows) return;
  uint64_t a, b;
  if (!decode_row(R, r, &a, &b) || (R.row_len && r + 1 < R.n_rows && R.row_ptr[r + 1] < R.row_ptr[r])) {
    if ((threadIdx.x & 31) == 0) { count[r] = 0; atomicOr(&ctl->err, DEC_ERR_ROWS); }
    return;
  }
  bool have_first = false;
  uint64_t total = 0;
  for (uint64_t k = a; k < b; k += 32) {
    const DecodeTok t = decode_step(T, R, k + (threadIdx.x & 31), b, skip != 0, &have_first);
    total += __reduce_add_sync(0xFFFFFFFFu, t.len);
  }
  if ((threadIdx.x & 31) == 0) {
    if (total >= DEC_MAX_ROW_TEXT) { atomicOr(&ctl->err, DEC_ERR_ROW_SIZE); total = 0; }
    count[r] = (uint32_t)total;
  }
}

// The emission window of one warp (D2): stage[i] is the byte of global address wbase + i (wbase 16-byte aligned), bytes
// [lo, fill) are staged and not yet stored.  flush stores them: whole 16-byte blocks as one uint4 per lane, the partial
// blocks at the window's edges byte by byte (their other bytes belong to the neighbouring row).  all = false keeps the
// partial last block staged and moves it to the front of the window.
struct EmitWindow { uint64_t wbase; uint32_t lo, fill; };
__device__ __forceinline__ void stage_flush(uint8_t* stage, uint8_t* text, EmitWindow& w, bool all) {
  const int lane = threadIdx.x & 31;
  const uint32_t end = all ? w.fill : (w.fill & ~15u);
  if (end > w.lo) {
    const uint32_t b0 = (w.lo + 15u) & ~15u, b1 = end & ~15u;
    const uint32_t head_end = b0 < end ? b0 : end;
    if (w.lo + lane < head_end) text[w.wbase + w.lo + lane] = stage[w.lo + lane];
    for (uint32_t j = b0 + 16u * lane; j + 16u <= b1; j += 512u)
      *reinterpret_cast<uint4*>(text + w.wbase + j) = *reinterpret_cast<const uint4*>(stage + j);
    if (b0 <= b1 && b1 + lane < end) text[w.wbase + b1 + lane] = stage[b1 + lane];
  }
  if (all) return;
  const uint32_t keep = w.fill & ~15u;
  if (keep <= w.lo) return;   // (nothing stored: the window is still inside its first block)
  __syncwarp();
  const uint8_t v = lane < (int)(w.fill - keep) ? stage[keep + lane] : 0;
  __syncwarp();
  if (lane < (int)(w.fill - keep)) stage[lane] = v;
  __syncwarp();
  w.wbase += keep; w.fill -= keep; w.lo = 0;
}

// D2: row r's images at text[off[r] ..), off[r] (and off[n_rows] by the last row) from the scan of D1's counts.  The
// 32-token steps are gathered into the warp's window, which is stored in whole 16-byte blocks when the next step does
// not fit it and at the row's end; a step whose images do not fit an empty window (over about 2 KB) is stored by each
// lane for its own token.  With lossy_count (ByteLevel): the row's length after
// from_utf8_lossy, and ctl->bad when it differs from the row's bytes.
__global__ void __launch_bounds__(DEC_THREADS) decode_emit_kernel(const DecodeTable T, const DecodeRows R, uint32_t skip, const uint32_t* __restrict__ count,
                                                                  const unsigned long long* __restrict__ lexcl, const unsigned long long* __restrict__ bsum,
                                                                  int scan_block, uint8_t* text, uint64_t* __restrict__ text_off,
                                                                  uint32_t* __restrict__ lossy_count, DecodeCtl* __restrict__ ctl) {
  __shared__ __align__(16) uint8_t s_stage[DEC_THREADS / 32][DEC_STAGE];
  const uint32_t r = (uint32_t)(((uint64_t)blockIdx.x * DEC_THREADS + threadIdx.x) >> 5);
  if (r >= R.n_rows) return;
  const int lane = threadIdx.x & 31;
  uint8_t* stage = s_stage[(threadIdx.x >> 5)];
  const uint64_t base = lexcl[r] + bsum[r / scan_block];
  if (lane == 0) { text_off[r] = base; if (r + 1 == R.n_rows) text_off[r + 1] = base + count[r]; }
  uint64_t a, b;
  decode_row(R, r, &a, &b);   // (D1 has checked it)
  bool have_first = false;
  uint64_t pos = base;
  EmitWindow w{base & ~15ull, (uint32_t)(base & 15u), (uint32_t)(base & 15u)};
  for (uint64_t k = a; k < b; k += 32) {
    const DecodeTok t = decode_step(T, R, k + lane, b, skip != 0, &have_first);
    const uint32_t incl = warp_incl_sum(t.len), step = __shfl_sync(0xFFFFFFFFu, incl, 31), ex = incl - t.len;
    const uint8_t* __restrict__ src = T.pool + t.off;
    if (w.fill + step > (uint32_t)DEC_STAGE) {   // the window is full: store its whole blocks, keep the partial last one
      stage_flush(stage, text, w, false);
      __syncwarp();
    }
    if (w.fill + step <= (uint32_t)DEC_STAGE) {
      for (uint32_t j = 0; j < t.len; ++j) stage[w.fill + ex + j] = __ldg(src + j);
      w.fill += step;
      __syncwarp();
    } else {   // a step of very long images: store what is staged, then each lane its own token, and restart the window
      stage_flush(stage, text, w, true);
      for (uint32_t j = 0; j < t.len; ++j) text[pos + ex + j] = __ldg(src + j);
      const uint64_t next = pos + step;
      w = EmitWindow{next & ~15ull, (uint32_t)(next & 15u), (uint32_t)(next & 15u)};
      __syncwarp();
    }
    pos += step;
  }
  stage_flush(stage, text, w, true);
  if (!lossy_count) return;
  __syncwarp();   // (the row's bytes, stored by the lanes of this warp, are read back below)
  // one byte per lane, consecutive lanes on consecutive bytes; an ASCII byte is valid without its neighbours.  (Reading
  // 16 bytes per lane and classifying the non-ASCII blocks with 16 lanes each took longer on the GPT-2 corpus, whose
  // text has a byte of 80-FF in many of its 16-byte blocks.)
  const uint8_t* row = text + base;
  const int64_t len = (int64_t)(pos - base);
  uint32_t out = 0, bad = 0;
  for (int64_t p = lane; p < len; p += 32) {
    const int c = row[p] < 0x80u ? LOSSY_VALID : lossy_class(row, p, len);
    out += lossy_bytes(c);
    bad |= c != LOSSY_VALID;
  }
  out = __reduce_add_sync(0xFFFFFFFFu, out);
  bad = __any_sync(0xFFFFFFFFu, bad);
  if (lane == 0) {
    lossy_count[r] = out;
    if (bad) atomicOr(&ctl->bad, 1u);
  }
}

// D3: row r of text (src_off) through from_utf8_lossy into out at the scan of D2's lossy counts; out_off as D2's text_off
__global__ void __launch_bounds__(DEC_THREADS) decode_lossy_kernel(const uint8_t* __restrict__ text, const uint64_t* __restrict__ src_off, uint32_t n_rows,
                                                                   const uint32_t* __restrict__ lossy_count, const unsigned long long* __restrict__ lexcl,
                                                                   const unsigned long long* __restrict__ bsum, int scan_block, uint8_t* __restrict__ out,
                                                                   uint64_t* __restrict__ out_off) {
  const uint32_t r = (uint32_t)(((uint64_t)blockIdx.x * DEC_THREADS + threadIdx.x) >> 5);
  if (r >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const uint64_t base = lexcl[r] + bsum[r / scan_block];
  if (lane == 0) { out_off[r] = base; if (r + 1 == n_rows) out_off[r + 1] = base + lossy_count[r]; }
  const uint8_t* row = text + src_off[r];
  const int64_t len = (int64_t)(src_off[r + 1] - src_off[r]);
  uint64_t pos = base;
  for (int64_t p0 = 0; p0 < len; p0 += 32) {
    const int64_t p = p0 + lane;
    const int c = p < len ? lossy_class(row, p, len) : LOSSY_SWALLOW;
    const uint32_t n = lossy_bytes(c), incl = warp_incl_sum(n), ex = incl - n;
    if (c == LOSSY_VALID) out[pos + ex] = row[p];
    else if (c == LOSSY_REPLACE) { out[pos + ex] = 0xEFu; out[pos + ex + 1] = 0xBFu; out[pos + ex + 2] = 0xBDu; }
    pos += __shfl_sync(0xFFFFFFFFu, incl, 31);
  }
}
#endif

}  // namespace b2t
