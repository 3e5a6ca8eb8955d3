// norm_kernels.cuh -- BertNormalizer on the device, as a byte-rewriting pre-pass in front of the scan kernels.
//
// Replaces (paths relative to tokenizers/src of huggingface/tokenizers):
//   normalizers/bert.rs:92-136          clean_text, handle_chinese_chars, strip_accents (NFD + drop Mn), lowercase
//   tokenizer/normalizer.rs:317-428     NormalizedString::transform: the alignment of every normalized character with
//                                       the original character it came from, which is what token offsets are made of
//
// Every step of BertNormalizer maps ONE character to a (possibly empty) sequence of characters without looking at its
// neighbours, so the whole normalizer is a table: code point -> UTF-8 bytes of its image (host_tables.cu composes it
// from the probed per-character facts of bert_tables.inc for the four flags).  The one context-dependent part of NFD,
// canonical reordering of combining marks, mostly permutes characters that strip_accents then drops: of the 817 characters
// whose NFD starts with a non-zero combining class all but 83 are removed (probed, tools/gen_bert_tables.py).  Order still
// matters for the alignment of the 83 survivors: NormalizedString hands the original characters out in input order, so a
// survivor that sorting moves past a mark -- in front of it or behind it, also one that clean_text removed between them --
// takes that mark's character.  A survivor with a neighbour that lets canonical ordering reach it is refused
// (norm_survivor_refused: ERR_NORM_UNSUPPORTED -> B2T_ERR_UNSUPPORTED), never aligned differently.
//
//   N1 norm_count   per 2 KB page of the ORIGINAL batch: bytes of its image, characters it holds
//   (exclusive scans of both, one host read of the total)
//   N2 norm_write   the normalized batch, and for every normalized byte the index of its ORIGINAL character (src_char);
//                   document offsets in the normalized batch + the original character index of every document start
//   ... the ordinary pipeline runs on the normalized batch with byte offsets ...
//   N3 norm_offsets token (byte_start, byte_end) in the normalized document -> (char_start, char_end) in the ORIGINAL
//                   one: [src_char(first byte), src_char(last byte) + 1) -- the union of the alignments of the token's
//                   first and last character, exactly what the reference reports (pre_tokenizer.rs:198-263 + normalizer.rs
//                   alignments; probed: a dropped accent or control character inside a token widens it, one behind it does not)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "b2t_tables.h"
#include "pretok_logic.cuh"

namespace b2t {

enum { ERR_NORM_UNSUPPORTED = 16u };
constexpr int NORM_THREADS = 256;
constexpr int NORM_PER_THREAD = PAGE / NORM_THREADS;   // 8 bytes

struct NormTables {
  const uint16_t* blk;      // [0x110000 >> 7]: block of the code point
  const uint32_t* ent;      // [blocks][128]: kind (bits 0-1) | flags | byte length (bits 2-6) | pool offset (bits 8-31), b2t_tables.h
  const uint8_t* pool;      // UTF-8 images
  const uint8_t* ascii;     // [128]: image of an ASCII character (always one ASCII character), 0xFF = dropped
};

__host__ __device__ inline uint32_t norm_entry(const NormTables& T, uint32_t cp) {
  return T.ent[(uint32_t)T.blk[cp >> 7] * 128u + (cp & 127u)];
}

// the character that starts at p (a lead byte): code point and byte length (bytes past the end read as 0)
__host__ __device__ inline uint32_t norm_decode(const uint8_t* b, int64_t p, int64_t n, int* len) {
  const uint32_t b0 = b[p];
  if (b0 < 0x80u) { *len = 1; return b0; }
  const int l = b0 < 0xE0u ? 2 : (b0 < 0xF0u ? 3 : 4);
  uint32_t cp = b0 & (0x7Fu >> l);
  for (int k = 1; k < l; ++k) cp = (cp << 6) | (p + k < n ? (b[p + k] & 0x3Fu) : 0u);
  *len = l;
  return cp < 0x110000u ? cp : 0x10FFFFu;
}

// The character at byte p of the batch bytes[0, n) is a survivor or keeps a mark behind its first piece (NORM_TAIL_FLAG):
// refused unless its image is itself (a survivor) and neither the character in front of it (a survivor) nor the one behind it
// lets canonical ordering reach its kept mark (norm_mark_neighbour).  Then NFD leaves the mark where it is -- behind the
// class-0 character before it, in front of anything it could change places with -- and NormalizedString aligns it with its
// own character, as the image table does.  The neighbours are read in the packed batch, so a mark at a document edge looks
// across it (a needless refusal at worst); the batch's ends stop the look.
__host__ __device__ inline bool norm_survivor_refused(const uint8_t* bytes, int64_t p, int64_t n, const NormTables& T, const uint8_t* ascii) {
  int len, l2;
  const uint32_t e = norm_entry(T, norm_decode(bytes, p, n, &len));
  if ((e & 3u) == NORM_SURVIVOR && (e & NORM_MARK_FLAG)) return true;
  if ((e & 3u) == NORM_SURVIVOR && p > 0) {
    int64_t q = p - 1;
    while (q > 0 && (bytes[q] & 0xC0u) == 0x80u && p - q < 4) --q;
    const uint32_t cp = norm_decode(bytes, q, n, &l2);
    if (norm_mark_neighbour(cp, norm_entry(T, cp), ascii)) return true;
  }
  if (p + len < n) {
    const uint32_t cp = norm_decode(bytes, p + len, n, &l2);
    if (norm_mark_neighbour(cp, norm_entry(T, cp), ascii)) return true;
  }
  return false;
}

// block-wide exclusive scan of one int per thread (256 threads); returns the exclusive prefix, *total = block sum
__device__ __forceinline__ int norm_block_scan(int v, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int s = 1; s < 32; s <<= 1) { const int o = __shfl_up_sync(0xFFFFFFFFu, inc, s); if (lane >= s) inc += o; }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  int base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < NORM_THREADS / 32; ++w) { const int x = s_warp[w]; if (w < warp) base += x; tot += x; }
  __syncthreads();
  *total = tot;
  return base + inc - v;
}

// What a thread learns about its 8 bytes: per byte the length of the image of the character that starts there
// (6 bits each, 63 = "not a character start"), the table entry of the non-ASCII ones is looked up again when writing.
constexpr uint32_t NORM_NOT_LEAD = 63u;
// An image is at most 3x its character (Hangul syllable -> three jamo; host_tables.cu checks every entry), and a page emits
// the whole image of its last character even if up to 3 of that character's bytes lie in the next page.
constexpr int NORM_MAX_OUT = 3 * (PAGE + 3) + 7;

struct NormChunk {
  uint32_t w0, w1, w2;     // the thread's 8 bytes and the 4 behind them (little endian)
  unsigned long long lens; // 8 x 6 bits
  uint32_t ent[NORM_PER_THREAD];   // table entry of the non-ASCII character that starts at byte i (0 otherwise)
  int n_out, n_chars;
};

__device__ __forceinline__ uint32_t norm_bytes_at(const NormChunk& c, int i) {   // the four bytes that start at byte i (i < 8)
  const uint32_t lo = i < 4 ? c.w0 : c.w1, hi = i < 4 ? c.w1 : c.w2;
  return __funnelshift_r(lo, hi, 8 * (i & 3));
}
__device__ __forceinline__ uint32_t norm_cp_of(uint32_t v, int* len) {           // v: the character's bytes, little endian
  const uint32_t b0 = v & 0xFFu;
  const int l = b0 < 0xE0u ? 2 : (b0 < 0xF0u ? 3 : 4);
  const uint32_t t24 = ((v & 0x3Fu) << 18) | ((v << 4) & 0x3F000u) | ((v >> 10) & 0xFC0u) | ((v >> 24) & 0x3Fu);
  uint32_t cp = (t24 >> (6 * (4 - l))) & ((2u << (5 * l)) - 1u);
  *len = l;
  return cp < 0x110000u ? cp : 0x10FFFFu;
}

// The table look-ups of a thread's (up to 8) non-ASCII characters are issued together -- first all block numbers, then all
// entries -- instead of one dependent pair per character: the pre-pass is bound by the latency of these loads.
__device__ __forceinline__ void norm_load_chunk(const uint8_t* __restrict__ bytes, int64_t n, int64_t base, const NormTables& T, const uint8_t* s_ascii,
                                                NormChunk& c, uint32_t* err) {
  c.w0 = c.w1 = c.w2 = 0u; c.lens = 0ull; c.n_out = 0; c.n_chars = 0;
#pragma unroll
  for (int i = 0; i < NORM_PER_THREAD; ++i) c.ent[i] = 0u;
  if (base >= n) { c.lens = ~0ull; return; }
  if (base + 12 <= n) {
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(bytes + base));
    c.w0 = v.x; c.w1 = v.y; c.w2 = __ldg(reinterpret_cast<const uint32_t*>(bytes + base + 8));
  } else {
    uint32_t w[3] = {0u, 0u, 0u};
    for (int k = 0; k < 12 && base + k < n; ++k) w[k >> 2] |= (uint32_t)__ldg(bytes + base + k) << (8 * (k & 3));
    c.w0 = w[0]; c.w1 = w[1]; c.w2 = w[2];
  }
  const int valid = n - base >= NORM_PER_THREAD ? NORM_PER_THREAD : (int)(n - base);
  uint32_t cps[NORM_PER_THREAD], clen[NORM_PER_THREAD], blk[NORM_PER_THREAD];
  uint32_t lead = 0u, hi = 0u, surv = 0u;   // bit i: byte i starts a character / a non-ASCII character / one with a kept mark
#pragma unroll
  for (int i = 0; i < NORM_PER_THREAD; ++i) {
    const uint32_t b0 = ((i < 4 ? c.w0 : c.w1) >> (8 * (i & 3))) & 0xFFu;
    int l = 1;
    cps[i] = b0;
    if (i < valid && (b0 & 0xC0u) != 0x80u) {
      lead |= 1u << i;
      if (b0 >= 0x80u) { hi |= 1u << i; cps[i] = norm_cp_of(norm_bytes_at(c, i), &l); }
    }
    clen[i] = (uint32_t)l;
  }
#pragma unroll
  for (int i = 0; i < NORM_PER_THREAD; ++i) blk[i] = (hi >> i) & 1u ? (uint32_t)__ldg(T.blk + (cps[i] >> 7)) : 0u;
#pragma unroll
  for (int i = 0; i < NORM_PER_THREAD; ++i) if ((hi >> i) & 1u) c.ent[i] = __ldg(T.ent + blk[i] * 128u + (cps[i] & 127u));
#pragma unroll
  for (int i = 0; i < NORM_PER_THREAD; ++i) {
    uint32_t len = NORM_NOT_LEAD;
    if ((lead >> i) & 1u) {
      ++c.n_chars;
      if (!((hi >> i) & 1u)) len = s_ascii[cps[i]] != 0xFFu ? 1u : 0u;
      else {
        const uint32_t e = c.ent[i], kind = e & 3u;
        len = kind == NORM_REMOVE ? 0u : (kind == NORM_STRING ? ((e >> 2) & NORM_LEN_MASK) : clen[i]);
        if (kind == NORM_SURVIVOR || (kind == NORM_STRING && (e & NORM_TAIL_FLAG))) surv |= 1u << i;
      }
      c.n_out += (int)len;
    }
    c.lens |= (unsigned long long)len << (6 * i);
  }
  // kept marks are rare: one copy of the check serves them all, outside the unrolled loop
  for (; surv; surv &= surv - 1u)
    if (norm_survivor_refused(bytes, base + __ffs(surv) - 1, n, T, s_ascii)) atomicOr(err, ERR_NORM_UNSUPPORTED);
}

// ------------------------------------------------------------------------------------------------ N1
__global__ void __launch_bounds__(NORM_THREADS, 8) norm_count_kernel(const uint8_t* __restrict__ bytes, int64_t n, const NormTables T,
                                                                  uint32_t* __restrict__ page_out, uint32_t* __restrict__ page_chars, uint32_t* __restrict__ err) {
  __shared__ int s_warp[NORM_THREADS / 32];
  __shared__ uint8_t s_ascii[128];
  if (threadIdx.x < 128) s_ascii[threadIdx.x] = __ldg(T.ascii + threadIdx.x);
  __syncthreads();
  NormChunk c;
  norm_load_chunk(bytes, n, (int64_t)blockIdx.x * PAGE + (int64_t)threadIdx.x * NORM_PER_THREAD, T, s_ascii, c, err);
  int tot_out, tot_chars;
  norm_block_scan(c.n_out, s_warp, &tot_out);
  norm_block_scan(c.n_chars, s_warp, &tot_chars);
  if (threadIdx.x == 0) { page_out[blockIdx.x] = (uint32_t)tot_out; page_chars[blockIdx.x] = (uint32_t)tot_chars; }
}

// ------------------------------------------------------------------------------------------------ N2
// out_lexcl / out_bexcl, chr_lexcl / chr_bexcl: exclusive scans of N1's counts (two-level: local + block, as the token-count
// scan).  The page's image is assembled in shared memory (bytes + page-relative original character index) and written out
// with consecutive threads on consecutive addresses.
__global__ void __launch_bounds__(NORM_THREADS, 6) norm_write_kernel(const uint8_t* __restrict__ bytes, int64_t n, const NormTables T,
                                                                  const unsigned long long* __restrict__ out_lexcl, const unsigned long long* __restrict__ out_bexcl,
                                                                  const unsigned long long* __restrict__ chr_lexcl, const unsigned long long* __restrict__ chr_bexcl, int scan_block,
                                                                  const uint32_t* __restrict__ page_first_doc, const uint64_t* __restrict__ doc_off, uint32_t n_docs,
                                                                  uint8_t* __restrict__ out, uint32_t* __restrict__ src_char,
                                                                  uint64_t* __restrict__ doc_off_out, uint32_t* __restrict__ doc_char0, uint32_t* __restrict__ err) {
  __shared__ int s_warp[NORM_THREADS / 32];
  __shared__ uint8_t s_ascii[128];
  __shared__ uint8_t s_img[NORM_MAX_OUT];
  __shared__ uint16_t s_src[NORM_MAX_OUT];
  __shared__ uint16_t s_oex[NORM_THREADS], s_cex[NORM_THREADS];
  __shared__ unsigned long long s_lens[NORM_THREADS];
  if (threadIdx.x < 128) s_ascii[threadIdx.x] = __ldg(T.ascii + threadIdx.x);
  __syncthreads();
  const int64_t t = blockIdx.x;
  const int64_t base = t * PAGE + (int64_t)threadIdx.x * NORM_PER_THREAD;
  // loads that depend on nothing computed here go first (the kernel is a chain of latencies: bytes -> table -> scans -> stores)
  const unsigned long long g_out = out_lexcl[t] + out_bexcl[t / scan_block], g_chr = chr_lexcl[t] + chr_bexcl[t / scan_block];
  const uint64_t d_first = (uint64_t)__ldg(page_first_doc + t) + threadIdx.x;
  const int64_t q_first = d_first <= n_docs ? (int64_t)__ldg(doc_off + d_first) : (int64_t)1 << 62;
  NormChunk c;
  norm_load_chunk(bytes, n, base, T, s_ascii, c, err);
  int tot_out, tot_chars;
  int o = norm_block_scan(c.n_out, s_warp, &tot_out);       // page-relative position in the image
  int ch = norm_block_scan(c.n_chars, s_warp, &tot_chars);  // page-relative character index
  // what the document pass below needs from every thread: where its 8 bytes start in the image / in characters, and the lengths
  s_oex[threadIdx.x] = (uint16_t)o; s_cex[threadIdx.x] = (uint16_t)ch; s_lens[threadIdx.x] = c.lens;
  // Emit byte by byte over the 8 bytes of the thread and the (up to 3) bytes behind them that finish its last character:
  // ASCII characters and non-ASCII characters whose image is themselves -- nearly everything -- are copied through by the
  // same few instructions in every lane; only a character with a table image (upper case, accents, CJK spacing) loops.
  {
    int copy = 0, chi = ch;
#pragma unroll
    for (int j = 0; j < NORM_PER_THREAD + 3; ++j) {
      const uint32_t b = ((j < 4 ? c.w0 : (j < 8 ? c.w1 : c.w2)) >> (8 * (j & 3))) & 0xFFu;
      if (j < NORM_PER_THREAD) {
        const uint32_t len = (uint32_t)(c.lens >> (6 * j)) & 63u;
        if (len != NORM_NOT_LEAD) {            // a character of this thread starts here
          const uint32_t e = c.ent[j];         // 0 for ASCII
          const bool str = (e & 3u) == NORM_STRING;
          chi = ch++;
          copy = (len != 0u && !str) ? 1 : 0;
          if (str) {
            const uint8_t* __restrict__ src = T.pool + (e >> 8);
            for (uint32_t k = 0; k < len; ++k) { s_img[o + k] = __ldg(src + k); s_src[o + k] = (uint16_t)chi; }
            o += (int)len;
          }
        }
      } else if ((b & 0xC0u) != 0x80u) copy = 0;   // behind the 8 bytes: only continuation bytes of the last character
      if (copy) { s_img[o] = b < 0x80u ? s_ascii[b] : (uint8_t)b; s_src[o] = (uint16_t)chi; ++o; }
    }
  }
  __syncthreads();
  // the documents that start in this page (consecutive from page_first_doc[t]; the last page also owns the end sentinel):
  // their start in the image and the index of their first original character
  {
    const int64_t page_lo = t * PAGE, page_hi = page_lo + PAGE;
    for (uint64_t d = d_first; d <= n_docs; d += NORM_THREADS) {
      const int64_t q = d == d_first ? q_first : (int64_t)__ldg(doc_off + d);
      if (q >= page_hi) break;
      if (q < page_lo) continue;       // (cannot happen: page_first_doc is the first document at or behind the page start)
      const int owner = (int)(q - page_lo) / NORM_PER_THREAD, within = (int)(q - page_lo) % NORM_PER_THREAD;
      int oo = s_oex[owner], cc = s_cex[owner];
      const unsigned long long lens = s_lens[owner];
      for (int i = 0; i < within; ++i) {
        const uint32_t len = (uint32_t)(lens >> (6 * i)) & 63u;
        if (len != NORM_NOT_LEAD) { oo += (int)len; ++cc; }
      }
      doc_off_out[d] = g_out + (unsigned long long)oo;
      doc_char0[d] = (uint32_t)(g_chr + (unsigned long long)cc);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < tot_out; i += NORM_THREADS) {
    out[g_out + i] = s_img[i];
    src_char[g_out + i] = (uint32_t)(g_chr + s_src[i]);
  }
}

// ------------------------------------------------------------------------------------------------ N3
// One warp per document: byte offsets in the normalized document -> character offsets in the original one.
__global__ void norm_offsets_kernel(const uint64_t* __restrict__ row_ptr, uint32_t n_docs, unsigned long long token_base,
                                    const uint64_t* __restrict__ doc_off_norm, const uint32_t* __restrict__ doc_char0,
                                    const uint32_t* __restrict__ src_char, uint2* __restrict__ offsets) {
  const uint32_t d = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (d >= n_docs) return;
  const uint64_t a = row_ptr[d] - token_base, b = row_ptr[d + 1] - token_base;
  const uint64_t base = doc_off_norm[d];
  const uint32_t c0 = doc_char0[d];
  for (uint64_t i = a + lane; i < b; i += 32) {
    const uint2 o = offsets[i];
    uint2 r = make_uint2(0u, 0u);
    if (o.y > o.x) r = make_uint2(__ldg(src_char + base + o.x) - c0, __ldg(src_char + base + o.y - 1) + 1u - c0);
    offsets[i] = r;
  }
}

}  // namespace b2t
