// long_kernels.cuh -- the path for BPE pre-tokens longer than LONG_PRETOK_MIN bytes (URLs, base64 blobs, 64 KB letter / space
// runs of the length-skew stress config).  They do not fit the per-page shared-memory scheme of model_kernels.cuh and
// would stall their page for milliseconds, so they are resolved by a pre-pass:
//   K1c long_find : one warp per page finds the pre-tokens that start in the page and are longer than LONG_PRETOK_MIN;
//       soft_cut  : cuts them wherever no token of the vocabulary can span the byte boundary (the two bytes are not a
//                   token and neither byte triple around the boundary occurs inside any token): merges never cross such a
//                   boundary, so the pieces are merged independently -- by the page kernel like ordinary pre-tokens when
//                   they are short (almost always), else by K2L.  The cuts live in a second bitmap (soft_bits): word ids and
//                   the split list of the reference are untouched;
//       long_find : (second pass, on start_bits | soft_bits) the pieces that are still longer than LONG_PRETOK_MIN get
//                   consecutive slots (page_long[page] = first slot) and a region of the long pool;
//   K2L bpe_long  : one block per long pre-token runs the merge loop of models/bpe/word.rs:162-250 on arrays in global
//                   memory and leaves the token list (id, end byte, char offsets relative to the pre-token) in the pool;
//   K2            : copies those tokens into the CSR at the right place (model_kernels.cuh).
// Merge order: the reference pops (rank, pos) from a heap; that equals "merge the leftmost pair of minimal rank" per
// round.  When the merge table is MONOTONE (every merge ranks after all merges that create its parts -- true for any
// trained BPE, checked at table build) all occurrences of the minimal-rank pair can be merged in the same round
// (left to right, non-overlapping), because nothing a merge creates can rank lower; that is what makes a 64 KB run
// take O(#distinct ranks) rounds instead of O(length).  Otherwise one merge per round.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "b2t_tables.h"
#include "pretok_logic.cuh"

namespace b2t {

constexpr int LONG_PRETOK_MIN = 256;       // pre-tokens with more bytes than this take the long path (== BPE halo of K2)
constexpr int LONG_THREADS = 1024;  // one block per long pre-token; 256 -> 1024 threads measured on the 64 KB runs of config 5
enum { ERR_POOL_OVERFLOW = 2u, ERR_INTERNAL = 4u };

struct LongCtl {        // device-side counters, zeroed per batch
  uint32_t n_long;      // number of long pieces after the soft cuts (second pass)
  uint32_t err;
  unsigned long long pool_used;  // bytes of long pieces placed (or wanted, on overflow) in the pool
  uint32_t n_long1;     // number of long pre-tokens before the cuts (first pass)
  uint32_t pad;
};

struct LongPool {
  uint32_t* id;     // symbol id at its start position
  uint64_t* val;    // rank << 32 | new_id of the pair (symbol at i, next symbol), NO_MERGE if none
  uint32_t* len;    // symbol length in bytes (0 = not a symbol start)
  uint32_t* plen;   // length of the previous symbol (to step left)
  uint32_t* aux;    // scratch for the block scans
  uint4* out;       // tokens: {id, end byte (relative), char start (relative), char end (relative)}
  unsigned long long cap;  // pool capacity in pre-token bytes
};

struct LongDesc {
  long long start, end;          // absolute byte range of the pre-token
  unsigned long long pool_off;   // its region of the pool
  uint32_t ntok;                 // filled by K2L
  uint32_t soft;                 // 1: a piece of a cut pre-token (the ignore_merges whole-word rule does not apply to it)
};

// ------------------------------------------------------------------------------------------------ K1c
// One warp per page.  A start bit at p begins a long pre-token iff no start bit lies in (p, p + LONG_PRETOK_MIN].
// PASS 0: on start_bits, fills desc (start, end) and ctl->n_long1.  PASS 1: on start_bits | soft_bits for the pages flagged
// in page_soft (all others get page_long = -1), fills desc with pool regions, ctl->n_long and page_long.
template <int PASS>
__global__ void long_find_kernel(const uint32_t* __restrict__ start_bits, const uint32_t* __restrict__ soft_bits,
                                 const uint8_t* __restrict__ page_soft, int64_t n, int64_t n_pages, LongCtl* ctl,
                                 LongDesc* desc, int32_t* __restrict__ page_long, unsigned long long pool_cap) {
  const int lane = threadIdx.x & 31;
  const int64_t page = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (page >= n_pages) return;
  if (PASS == 1 && !__ldg(page_soft + page)) { if (lane == 0) page_long[page] = -1; return; }
  const int64_t n_words = n / 32 + 1;
  const int64_t w0 = page * (PAGE / 32);
  static_assert(PAGE / 32 == 64, "a lane handles words lane and lane + 32 of the page");
  constexpr int LW = LONG_PRETOK_MIN / 32;      // 8
  auto bits_at = [&](int64_t w) -> uint32_t {
    if (w >= n_words) return 0u;
    uint32_t b = __ldg(start_bits + w);
    if (PASS == 1) b |= __ldg(soft_bits + w);
    return b;
  };
  // lane handles words lane and lane + 32 of the page
  long long ps[2], qs[2];
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int64_t w = w0 + lane + half * 32;
    const uint32_t bits = bits_at(w);
    ps[half] = -1; qs[half] = -1;
    if (bits) {
      const int h = 31 - __clz((int)bits);
      bool is_long = true;
      for (int k = 1; k < LW && is_long; ++k)
        if (bits_at(w + k)) is_long = false;
      if (is_long && (bits_at(w + LW) & (h >= 31 ? 0xFFFFFFFFu : ((2u << h) - 1u)))) is_long = false;
      const long long p = w * 32 + h;
      if (is_long && p + LONG_PRETOK_MIN < n) {
        // find the end: first start bit after p + LONG_PRETOK_MIN, or n
        long long q = -1;
        int64_t ww = w + LW;
        uint32_t b = bits_at(ww) & ~(h >= 31 ? 0xFFFFFFFFu : ((2u << h) - 1u));
        while (true) {
          if (b) { q = ww * 32 + (__ffs((int)b) - 1); break; }
          ++ww;
          if (ww >= n_words) { q = n; break; }
          b = bits_at(ww);
        }
        if (q > n) q = n;
        ps[half] = p; qs[half] = q;
      }
    }
  }
  // slots in position order: all "half 0" words precede all "half 1" words of the page
  const unsigned m0 = __ballot_sync(0xFFFFFFFFu, ps[0] >= 0), m1 = __ballot_sync(0xFFFFFFFFu, ps[1] >= 0);
  const int total = __popc(m0) + __popc(m1);
  int base = 0;
  if (lane == 0) {
    if (PASS == 1) page_long[page] = -1;
    if (total) {
      base = (int)atomicAdd(PASS == 0 ? &ctl->n_long1 : &ctl->n_long, (uint32_t)total);
      if (PASS == 1) page_long[page] = base;
    }
  }
  base = __shfl_sync(0xFFFFFFFFu, base, 0);
  if (!total) return;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    if (ps[half] < 0) continue;
    const int slot = base + (half ? __popc(m0) + __popc(m1 & ((1u << lane) - 1u)) : __popc(m0 & ((1u << lane) - 1u)));
    LongDesc d;
    d.start = ps[half]; d.end = qs[half]; d.pool_off = 0; d.ntok = 0; d.soft = 0;
    if (PASS == 1) {
      const unsigned long long L = (unsigned long long)(qs[half] - ps[half]);
      const unsigned long long off = atomicAdd(&ctl->pool_used, L);
      d.pool_off = off;
      if (off + L > pool_cap) { atomicOr(&ctl->err, ERR_POOL_OVERFLOW); d.pool_off = ~0ull; }
      // a piece of a cut pre-token starts or ends at a soft bit
      const bool real_s = (__ldg(start_bits + (d.start >> 5)) >> (d.start & 31)) & 1u;
      const bool real_e = d.end >= n || ((__ldg(start_bits + (d.end >> 5)) >> (d.end & 31)) & 1u);
      d.soft = (real_s && real_e) ? 0u : 1u;
    }
    desc[slot] = d;
  }
}

// One block per long pre-token of the first pass: bit i of soft_bits is set iff a cut before byte i is exact, i.e. no
// vocabulary token can contain bytes i-1 and i of this text next to each other:
//   the two bytes are not a token, the triple (i-2, i-1, i) occurs in no token, the triple (i-1, i, i+1) occurs in no token
// (a token of 2 bytes spanning the boundary IS that pair; a longer one contains one of the two triples; triples that
// would reach outside the pre-token cannot occur).  Every page the pre-token touches is flagged in page_soft.
__global__ void __launch_bounds__(256) soft_cut_kernel(const uint8_t* __restrict__ bytes, const LongCtl* __restrict__ ctl,
                                                       const LongDesc* __restrict__ desc, uint32_t* __restrict__ soft_bits,
                                                       uint8_t* __restrict__ page_soft, DeviceTables t) {
  const uint32_t n_long = ctl->n_long1;
  const int lane = threadIdx.x & 31;
  for (uint32_t j = blockIdx.x; j < n_long; j += gridDim.x) {
    const long long s = desc[j].start, e = desc[j].end;
    for (long long pg = s / PAGE + threadIdx.x; pg <= (e - 1) / PAGE; pg += blockDim.x) page_soft[pg] = 1;
    // a warp takes 32 consecutive positions (aligned to the bitmap words)
    for (long long w = (s >> 5) + (threadIdx.x >> 5); w * 32 < e; w += blockDim.x >> 5) {
      const long long i = w * 32 + lane;
      bool cut = false;
      if (i > s && i < e) {
        const uint32_t b1 = __ldg(bytes + i - 1), b2 = __ldg(bytes + i);
        const uint32_t k2 = b1 | (b2 << 8);
        cut = !((__ldg(t.tok2_bits + (k2 >> 5)) >> (k2 & 31)) & 1u);
        if (cut && i - 2 >= s) {
          const uint32_t k3 = __ldg(bytes + i - 2) | (b1 << 8) | (b2 << 16);
          cut = !((__ldg(t.tri_bits + (k3 >> 5)) >> (k3 & 31)) & 1u);
        }
        if (cut && i + 1 < e) {
          const uint32_t k3 = b1 | (b2 << 8) | (__ldg(bytes + i + 1) << 16);
          cut = !((__ldg(t.tri_bits + (k3 >> 5)) >> (k3 & 31)) & 1u);
        }
      }
      const unsigned m = __ballot_sync(0xFFFFFFFFu, cut);
      if (lane == 0 && m) atomicOr(soft_bits + w, m);
    }
  }
}

// ------------------------------------------------------------------------------------------------ K2L helpers
// Block-wide inclusive scan of arr[0..L) in place (global memory), op = max or sum.  Each thread owns a contiguous
// segment; two passes.
template <bool IS_MAX>
__device__ __forceinline__ void block_scan_inplace(uint32_t* arr, long long L, uint32_t* s_part) {
  const int tid = threadIdx.x;
  const long long seg = (L + LONG_THREADS - 1) / LONG_THREADS;
  const long long lo = (long long)tid * seg, hi = lo + seg < L ? lo + seg : L;
  uint32_t acc = 0;
  for (long long i = lo; i < hi; ++i) { uint32_t v = arr[i]; acc = IS_MAX ? (v > acc ? v : acc) : acc + v; arr[i] = acc; }
  s_part[tid] = acc;
  __syncthreads();
  // exclusive scan over the LONG_THREADS partials (Hillis-Steele)
  uint32_t v = acc;
  for (int s = 1; s < LONG_THREADS; s <<= 1) {
    uint32_t o = tid >= s ? s_part[tid - s] : 0u;
    __syncthreads();
    v = IS_MAX ? (o > v ? o : v) : v + o;
    s_part[tid] = v;
    __syncthreads();
  }
  const uint32_t carry = tid ? s_part[tid - 1] : 0u;
  __syncthreads();
  if (carry) for (long long i = lo; i < hi; ++i) { uint32_t x = arr[i]; arr[i] = IS_MAX ? (carry > x ? carry : x) : x + carry; }
  __syncthreads();
}

__device__ __forceinline__ uint64_t long_merge_lookup(const DeviceTables& t, uint32_t a, uint32_t b) {
  uint32_t h = pair_hash(a, b) & t.merge_mask;
  while (true) {
    uint4 e = __ldg(t.merge_tbl + h);
    if (e.x == a && e.y == b) return ((uint64_t)e.z << 32) | e.w;
    if (e.x == EMPTY_KEY) return NO_MERGE;
    h = (h + 1) & t.merge_mask;
  }
}

// ------------------------------------------------------------------------------------------------ K2L
__global__ void __launch_bounds__(LONG_THREADS) bpe_long_kernel(const uint8_t* __restrict__ bytes, const LongCtl* ctl, LongDesc* desc,
                                                                LongPool pool, DeviceTables t, int monotone) {
  __shared__ uint32_t s_part[LONG_THREADS];
  __shared__ unsigned long long s_red[LONG_THREADS / 32];
  __shared__ unsigned long long s_best;
  __shared__ int s_hit;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t n_long = ctl->n_long;
  for (uint32_t j = blockIdx.x; j < n_long; j += gridDim.x) {
    LongDesc d = desc[j];
    if (d.pool_off == ~0ull) continue;  // pool overflow: the host grows the pool and reruns
    const long long L = d.end - d.start;
    const uint8_t* __restrict__ src = bytes + d.start;
    uint32_t* id = pool.id + d.pool_off;
    uint64_t* val = pool.val + d.pool_off;
    uint32_t* len = pool.len + d.pool_off;
    uint32_t* plen = pool.plen + d.pool_off;
    uint32_t* aux = pool.aux + d.pool_off;
    uint4* out = pool.out + d.pool_off;

    // whole pre-token in the vocabulary (ignore_merges)?  The table holds every token, whatever its length (pieces of a
    // cut pre-token are never looked up).
    if (tid == 0) s_hit = 0;
    __syncthreads();
    if (t.ignore_merges && !d.soft && L < 65536 && tid == 0) {
      StrHash h; strhash_init(h);
      for (long long i = 0; i < L; ++i) strhash_byte(h, __ldg(src + i));
      strhash_fin(h);
      uint32_t slot = h.h1 & t.word_mask;
      while (true) {
        uint4 en = __ldg(t.word_tbl + slot);
        if (en.z == EMPTY_KEY) break;
        if (en.x == h.h2 && en.y == (uint32_t)L) {
          const uint8_t* q = t.word_pool + en.w;
          bool same = true;
          for (long long i = 0; i < L; ++i) if (__ldg(q + i) != __ldg(src + i)) { same = false; break; }
          if (same) { s_hit = 1; id[0] = en.z; break; }
        }
        slot = (slot + 1) & t.word_mask;
      }
    }
    __syncthreads();
    const bool hit = s_hit != 0;
    // ---- init symbols (one per byte)
    for (long long i = tid; i < L; i += LONG_THREADS) {
      if (!hit) id[i] = __ldg(t.byte_to_id + __ldg(src + i));
      len[i] = hit ? (i == 0 ? (uint32_t)L : 0u) : 1u;
      plen[i] = 1u;
    }
    __syncthreads();
    if (!hit) {
      for (long long i = tid; i < L; i += LONG_THREADS) val[i] = i + 1 < L ? long_merge_lookup(t, id[i], id[i + 1]) : NO_MERGE;
      __syncthreads();
      // ---- merge rounds
      while (true) {
        // leftmost pair of minimal rank: minimise (rank << 32 | pos) -- positions fit 31 bits
        unsigned long long best = ~0ull;
        for (long long i = tid; i < L; i += LONG_THREADS) {
          if (len[i]) {
            uint64_t v = val[i];
            if (v != NO_MERGE) {
              unsigned long long key = (v & 0xFFFFFFFF00000000ull) | (unsigned long long)i;
              if (key < best) best = key;
            }
          }
        }
#pragma unroll
        for (int s = 16; s >= 1; s >>= 1) { unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, best, s); best = o < best ? o : best; }
        if (lane == 0) s_red[warp] = best;
        __syncthreads();
        if (tid == 0) {
          unsigned long long b = s_red[0];
          for (int w = 1; w < LONG_THREADS / 32; ++w) b = s_red[w] < b ? s_red[w] : b;
          s_best = b;
        }
        __syncthreads();
        best = s_best;
        if (best == ~0ull) break;
        const uint32_t minrank = (uint32_t)(best >> 32);
        const long long minpos = (long long)(best & 0xFFFFFFFFull);
        const uint32_t newid = (uint32_t)val[minpos];
        const uint32_t x = id[minpos], xlen = len[minpos];
        const uint32_t y = id[minpos + xlen];
        __syncthreads();  // everyone has read the winner before anything is modified
        if (!monotone) {
          if (tid == 0) {
            const long long i = minpos, q = i + len[i];
            const uint32_t nl = len[i] + len[q];
            id[i] = newid; len[i] = nl; len[q] = 0;
            const long long nx = i + nl;
            if (nx < L) plen[nx] = nl;
            val[i] = nx < L ? long_merge_lookup(t, newid, id[nx]) : NO_MERGE;
            if (i > 0) { const long long pv = i - plen[i]; val[pv] = long_merge_lookup(t, id[pv], newid); }
          }
          __syncthreads();
          continue;
        }
        // monotone: merge every (non-overlapping, left to right) occurrence of the minimal-rank pair
        if (x == y) {
          // runs of x: occurrence k of a run merges iff k is even.  Run start via a max-scan of marker positions.
          for (long long i = tid; i < L; i += LONG_THREADS) {
            uint32_t g = 0;
            if (len[i]) {
              const bool cand = (uint32_t)(val[i] >> 32) == minrank;
              bool starts = true;  // not a candidate, or a candidate whose left neighbour is not one
              if (cand && i > 0) { const long long pv = i - plen[i]; starts = (uint32_t)(val[pv] >> 32) != minrank; }
              if (starts) g = (uint32_t)i + 1u;
            }
            aux[i] = g;
          }
          __syncthreads();
          block_scan_inplace<true>(aux, L, s_part);
        }
        // phase 1: merge (positions that merge never overlap)
        for (long long i = tid; i < L; i += LONG_THREADS) {
          if (!len[i] || (uint32_t)(val[i] >> 32) != minrank) continue;
          if (x == y) {
            const long long cs = (long long)aux[i] - 1;
            if (((i - cs) / xlen) & 1) continue;  // odd occurrence of its run: consumed by the merge to its left
          }
          const long long q = i + xlen;
          // an even occurrence whose right neighbour is the last x of the run is fine; but make sure q is still x's pair
          id[i] = newid; len[i] = xlen + len[q]; val[i] = NO_MERGE - 1;  // marker: merged this round
        }
        __syncthreads();
        // phase 2: kill the right halves, fix plen of the following symbol
        for (long long i = tid; i < L; i += LONG_THREADS) {
          if (len[i] && val[i] == NO_MERGE - 1) {
            const long long q = i + xlen;
            len[q] = 0;
            const long long nx = i + len[i];
            if (nx < L) plen[nx] = len[i];
          }
        }
        __syncthreads();
        // phase 3: ranks of the pairs around every merged symbol
        for (long long i = tid; i < L; i += LONG_THREADS) {
          if (len[i] && val[i] == NO_MERGE - 1) {
            const long long nx = i + len[i];
            if (i > 0) {
              const long long pv = i - plen[i];
              if (val[pv] != NO_MERGE - 1) val[pv] = long_merge_lookup(t, id[pv], newid);
            }
            aux[i] = nx < L ? 1u : 0u;  // remember: own rank still to be computed
          }
        }
        __syncthreads();
        for (long long i = tid; i < L; i += LONG_THREADS) {
          if (len[i] && val[i] == NO_MERGE - 1) {
            const long long nx = i + len[i];
            val[i] = nx < L ? long_merge_lookup(t, newid, id[nx]) : NO_MERGE;
          }
        }
        __syncthreads();
      }
    }
    // ---- token list: order = position order of the surviving symbols
    for (long long i = tid; i < L; i += LONG_THREADS) aux[i] = len[i] ? 1u : 0u;
    __syncthreads();
    block_scan_inplace<false>(aux, L, s_part);           // aux[i] = tokens in [0, i]
    const uint32_t ntok = aux[L - 1];
    // lead-byte prefix (chars) into plen (no longer needed)
    for (long long i = tid; i < L; i += LONG_THREADS) plen[i] = ((__ldg(src + i) & 0xC0u) != 0x80u) ? 1u : 0u;
    __syncthreads();
    block_scan_inplace<false>(plen, L, s_part);          // plen[i] = chars started in [0, i]
    for (long long i = tid; i < L; i += LONG_THREADS) {
      if (len[i]) {
        const long long e = i + len[i];
        out[aux[i] - 1] = make_uint4(id[i], (uint32_t)e, plen[i] - 1u, plen[e - 1]);
      }
    }
    if (tid == 0) desc[j].ntok = ntok;
    __syncthreads();
  }
}

}  // namespace b2t
