// pretok_kernels.cuh -- K0 doc_mark, K1 pre-tokenization scan (pretok_lean_kernel / pretok_stream_kernel, the
// HBM-roofline-graded kernel), K1b page_scan.
//
// Data layout in HBM (one batch = `n` packed UTF-8 bytes, documents back to back):
//   bytes      u8 [n]                input, read once by K1 with 16-byte loads
//   doc_bits   u32[n/32 + 2]         bit p set <=> some document starts at byte p (K0; bit n is the end sentinel)
//   start_bits u32[n/32 + 2]         bit p set <=> a pre-token (split) starts at byte p            (K1 output)
//   drop_bits  u32[n/32 + 2]         Whitespace / Bert: the split starting at p is removed whitespace (K1 output)
//   page_sum   u64[n/2048 + 1]       per 2 KB page: #chars, #kept splits, and the same counted from the last doc start
//   page_carry u64[n/2048 + 1]       K1b: #chars (low 32) / #kept splits (high 32) of the document that spans into the
//                                    page, counted from that document's start to the page start
//   page_first_doc u32[n/2048 + 1]   K0: first document d with doc_off[d] >= page start
// K1 algorithmic traffic: n bytes in + n/8 (doc_bits) in + n/8 (start_bits) out = 1.25 B per input byte.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "pretok_logic.cuh"

namespace b2t {

// ------------------------------------------------------------------------------------------------ K0
// One thread per document boundary d in [0, n_docs]: marks the doc start bit and fills page_first_doc.
__global__ void doc_mark_kernel(const uint64_t* __restrict__ doc_off, uint32_t n_docs, uint32_t* __restrict__ doc_bits,
                                uint32_t* __restrict__ page_first_doc) {
  uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d > n_docs) return;
  uint64_t pos = doc_off[d];
  atomicOr(&doc_bits[pos >> 5], 1u << (pos & 31));
  uint64_t p_hi = pos / PAGE;
  uint64_t p_lo = (d == 0) ? 0 : doc_off[d - 1] / PAGE + 1;
  for (uint64_t p = p_lo; p <= p_hi; ++p) page_first_doc[p] = d;
}

// ------------------------------------------------------------------------------------------------ K1 page summary
// page summary packing: [11:0] chars, [23:12] kept splits, [35:24] chars since last doc start, [47:36] splits since, [48] has doc start
__device__ __forceinline__ uint64_t pack_sum(uint32_t tot, uint32_t aft, uint32_t flag) {
  // tot / aft carry two 16-bit fields each (chars | splits << 16)
  return (uint64_t)(tot & 0xFFFu) | ((uint64_t)((tot >> 16) & 0xFFFu) << 12) | ((uint64_t)(aft & 0xFFFu) << 24) |
         ((uint64_t)((aft >> 16) & 0xFFFu) << 36) | ((uint64_t)(flag & 1u) << 48);
}

// ------------------------------------------------------------------------------------------------ K1b
// Exclusive SEGMENTED scan over the page summaries (segments restart at document starts) -> page_carry.
// Two tiny kernels: (1) every block scans 1024 pages (one per thread, coalesced) and emits its block summary,
// (2) one block scans the block summaries.  A page whose block has no document start before it adds its block's
// carry when it is consumed (bit 31 of the low word says "already absolute").
__device__ __forceinline__ void sum_unpack(uint64_t s, uint32_t& tc, uint32_t& ts, uint32_t& ac, uint32_t& as, uint32_t& f) {
  tc = (uint32_t)(s & 0xFFFu); ts = (uint32_t)((s >> 12) & 0xFFFu); ac = (uint32_t)((s >> 24) & 0xFFFu);
  as = (uint32_t)((s >> 36) & 0xFFFu); f = (uint32_t)((s >> 48) & 1u);
}

struct SegVal { uint32_t f, c, s; };  // "carry after" as a function of "carry before": f ? (c, s) : before + (c, s)
__device__ __forceinline__ SegVal seg_combine(SegVal earlier, SegVal later) {
  SegVal r;
  r.f = earlier.f | later.f;
  r.c = later.f ? later.c : earlier.c + later.c;
  r.s = later.f ? later.s : earlier.s + later.s;
  return r;
}
// inclusive block scan (1024 threads); returns this thread's inclusive value, *excl = exclusive value
__device__ __forceinline__ SegVal seg_block_scan(SegVal v, SegVal* excl, SegVal* s_w /*32*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int st = 1; st < 32; st <<= 1) {
    SegVal o;
    o.f = __shfl_up_sync(0xFFFFFFFFu, v.f, st); o.c = __shfl_up_sync(0xFFFFFFFFu, v.c, st); o.s = __shfl_up_sync(0xFFFFFFFFu, v.s, st);
    if (lane >= st) v = seg_combine(o, v);
  }
  if (lane == 31) s_w[warp] = v;
  __syncthreads();
  if (warp == 0) {
    SegVal w = s_w[lane];
#pragma unroll
    for (int st = 1; st < 32; st <<= 1) {
      SegVal o;
      o.f = __shfl_up_sync(0xFFFFFFFFu, w.f, st); o.c = __shfl_up_sync(0xFFFFFFFFu, w.c, st); o.s = __shfl_up_sync(0xFFFFFFFFu, w.s, st);
      if (lane >= st) w = seg_combine(o, w);
    }
    s_w[lane] = w;  // inclusive over warps
  }
  __syncthreads();
  SegVal before; before.f = 0; before.c = 0; before.s = 0;
  if (warp > 0) before = s_w[warp - 1];
  SegVal incl = seg_combine(before, v);
  SegVal pv;
  pv.f = __shfl_up_sync(0xFFFFFFFFu, v.f, 1); pv.c = __shfl_up_sync(0xFFFFFFFFu, v.c, 1); pv.s = __shfl_up_sync(0xFFFFFFFFu, v.s, 1);
  *excl = lane == 0 ? before : seg_combine(before, pv);
  __syncthreads();
  return incl;
}

constexpr int SCAN_BLOCK = 1024;

__global__ void __launch_bounds__(SCAN_BLOCK) page_scan_block_kernel(const uint64_t* __restrict__ page_sum, uint64_t* __restrict__ page_carry,
                                                                    uint64_t* __restrict__ block_sum, int64_t n_pages) {
  __shared__ SegVal s_w[32];
  const int64_t i = (int64_t)blockIdx.x * SCAN_BLOCK + threadIdx.x;
  SegVal v; v.f = 0; v.c = 0; v.s = 0;
  if (i < n_pages) {
    uint32_t tc, ts, ac, as, f;
    sum_unpack(__ldg(page_sum + i), tc, ts, ac, as, f);
    v.f = f; v.c = f ? ac : tc; v.s = f ? as : ts;
  }
  SegVal ex;
  SegVal incl = seg_block_scan(v, &ex, s_w);
  if (i < n_pages) page_carry[i] = (uint64_t)(ex.c | (ex.f << 31)) | ((uint64_t)ex.s << 32);
  if (threadIdx.x == SCAN_BLOCK - 1) block_sum[blockIdx.x] = (uint64_t)(incl.c | (incl.f << 31)) | ((uint64_t)incl.s << 32);
}

__global__ void __launch_bounds__(SCAN_BLOCK) page_scan_top_kernel(const uint64_t* __restrict__ block_sum, uint64_t* __restrict__ block_carry,
                                                                  int64_t n_blocks) {
  __shared__ SegVal s_w[32];
  __shared__ SegVal s_run;
  if (threadIdx.x == 0) { s_run.f = 0; s_run.c = 0; s_run.s = 0; }
  __syncthreads();
  for (int64_t base = 0; base < n_blocks; base += SCAN_BLOCK) {
    const int64_t i = base + threadIdx.x;
    SegVal v; v.f = 0; v.c = 0; v.s = 0;
    if (i < n_blocks) { uint64_t x = __ldg(block_sum + i); v.f = (uint32_t)(x >> 31) & 1u; v.c = (uint32_t)x & 0x7FFFFFFFu; v.s = (uint32_t)(x >> 32); }
    SegVal ex;
    SegVal incl = seg_block_scan(v, &ex, s_w);
    const SegVal run = s_run;
    const SegVal ex_abs = seg_combine(run, ex);
    if (i < n_blocks) block_carry[i] = (uint64_t)ex_abs.c | ((uint64_t)ex_abs.s << 32);
    __syncthreads();
    if (threadIdx.x == SCAN_BLOCK - 1) s_run = seg_combine(run, incl);
    __syncthreads();
  }
}

}  // namespace b2t

// ================================================================================================ K1
// pretok_lean_kernel (GPT-2, Whitespace, Bert, no regex) and pretok_stream_kernel (Llama-3), one kernel per
// pre-tokenizer with the same streaming structure.  Every WARP streams through its own contiguous range of the batch, 1 KB
// (32 chunks of 32 bytes, one per lane) per iteration, and is independent of all other warps: no shared memory, no
// block barrier.  Iteration i+1 is classified (pretok_logic.cuh: bit planes -> classes) before the boundaries of
// iteration i are evaluated, so a lane gets everything it needs from its neighbours with warp shuffles:
//   the chunk before lane 0   = lane 31 of the previous iteration (still in that lane's registers),
//   the chunk after lane 31   = lane 0 of the next iteration (already classified).
// The range ends are handled by classifying one extra KB on either side.  Page summaries (2 KB = two iterations of the
// same warp) are combined in registers.  Algorithmic traffic is unchanged: 1.25 B per input byte.
// Both kernels are built from the same steps (warp range, chunk load, valid mask, page summary); their loops stay
// apart because their register budgets and pipelines differ: the lean kernel runs at 64 registers, the Llama-3 kernel
// keeps two iterations of class masks live at 128.
namespace b2t {

constexpr int K1_THREADS = 128;
constexpr int K1_LEAN_MINBLOCKS = 8;
constexpr int K1_WINDOW_MINBLOCKS = 4;   // window (Llama-3) form: more live state

// ---------------------------------------------------------------------------------------------- steps of both kernels
// This warp's iterations [it_lo, it_hi); false when it has none.  it_lo is even: a page is two consecutive iterations
// of one warp.
__device__ __forceinline__ bool warp_range(int n_kb, int kb_per_warp, int& it_lo, int& it_hi) {
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  it_lo = gw * kb_per_warp;
  if (it_lo >= n_kb) return false;
  it_hi = it_lo + kb_per_warp < n_kb ? it_lo + kb_per_warp : n_kb;
  return true;
}

// the 32 bytes at p as little-endian words: two 16-byte loads
__device__ __forceinline__ void load32(const uint8_t* p, uint32_t w[8]) {
  const uint4* q = reinterpret_cast<const uint4*>(p);
  const uint4 a = __ldg(q), b = __ldg(q + 1);
  w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
}
// The chunk that holds the end of the batch: aligned word loads, bytes at or past n masked off.
__device__ __forceinline__ void load_tail_words(const uint8_t* bytes, uint32_t base, uint32_t n, uint32_t w[8]) {
  const uint32_t* __restrict__ words = reinterpret_cast<const uint32_t*>(bytes + base);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t p = base + 4u * j;
    uint32_t x = 0u;
    if (p < n) {
      x = __ldg(words + j);
      if (n - p < 4u) x &= (1u << (8u * (n - p))) - 1u;
    }
    w[j] = x;
  }
}
// load(it, w): the words of this lane's chunk of iteration `it` (it < 0: nothing there, all zero); bytes at or past n
// read as 0.  (A functor rather than a function: nvcc then lays out the lean kernel exactly as with a local lambda.)
struct ChunkLoader {
  const uint8_t* __restrict__ bytes;
  uint32_t n;
  int lane;
  __device__ __forceinline__ void operator()(int it, uint32_t w[8]) const {
    const uint32_t base = ((uint32_t)it * 32u + lane) * CHUNK;
    if (it >= 0 && base + CHUNK <= n) {
      load32(bytes + base, w);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) w[j] = 0u;
      if (it >= 0 && base < n) load_tail_words(bytes, base, n, w);
    }
  }
};
// the bytes of the chunk at `base` that lie inside the batch (none unless `there`)
__device__ __forceinline__ uint32_t chunk_valid(bool there, uint32_t base, uint32_t n) {
  return !there || base >= n ? 0u : (n - base >= CHUNK ? 0xFFFFFFFFu : (0xFFFFFFFFu >> (32u - (n - base))));
}

// The segmented page summary of a warp (counts restart at the last doc start of the page), built one iteration (half a
// page) at a time: add() takes this lane's lead bytes, kept splits and document starts of iteration `it`, and lane 0
// writes page_sum when the page is complete.  tot / aft / flag: the first half of the current page.
struct PageSummary {
  uint32_t tot, aft, flag;
  __device__ __forceinline__ void add(int it, int n_kb, uint32_t n, int lane, uint32_t lead, uint32_t kept, uint32_t docw,
                                      uint64_t* page_sum) {
    constexpr unsigned FULL = 0xFFFFFFFFu;
    const uint32_t t1 = (uint32_t)__popc(lead) | ((uint32_t)__popc(kept) << 16);
    const unsigned dsm = __ballot_sync(FULL, docw != 0u);
    const uint32_t wtot = __reduce_add_sync(FULL, t1);
    uint32_t waft = 0u;
    if (dsm) {
      const int last = 31 - __clz((int)dsm);
      uint32_t mine = 0u;
      if (lane > last) mine = t1;
      else if (lane == last) {
        const uint32_t from = ~bits_below(31 - __clz((int)docw));
        mine = (uint32_t)__popc(lead & from) | ((uint32_t)__popc(kept & from) << 16);
      }
      waft = __reduce_add_sync(FULL, mine);
    }
    const uint32_t wflag = dsm != 0u;
    const uint32_t page = (uint32_t)it >> 1;
    if (it & 1) {
      const uint32_t a = wflag ? waft : aft + wtot, t = tot + wtot, f = flag | wflag;
      if (lane == 0 && page * (uint32_t)PAGE <= n) page_sum[page] = pack_sum(t, a, f);
    } else {
      tot = wtot; aft = waft; flag = wflag;
      if (it + 1 >= n_kb && lane == 0 && page * (uint32_t)PAGE <= n) page_sum[page] = pack_sum(tot, aft, flag);  // the batch ends in the first half
    }
  }
};

// the four bytes at q..q+3 (q < n) as one word: two aligned loads and a funnel shift
struct At4Global {
  const uint32_t* __restrict__ words;
  uint32_t n;
  __device__ __forceinline__ uint32_t operator()(uint32_t q) const {
    const uint32_t a0 = __ldg(words + (q >> 2)), a1 = ((q | 3u) + 1u < n) ? __ldg(words + (q >> 2) + 1) : 0u;
    return __funnelshift_r(a0, a1, (q & 3u) * 8u);
  }
};

// ---------------------------------------------------------------------------------------------- lean form (GPT-2, Whitespace, no regex)
// Stage A (iteration j): bit planes, classes, and all of the boundary algebra that looks backwards.  Stage B
// (iteration j - 1): the one bit that looks forwards (finalize_gpt2), the store and the page summary.  Between the two
// a lane keeps six words, so the kernel runs at 64 registers.  There is one copy of the code: the loop starts one
// iteration before the warp's range (its output is discarded, only the carries are kept).
// ADDED: the batch went through the added-token extraction (added_kernels.cuh): the regex sees hard_bits (document starts +
// span boundaries) where it otherwise sees doc_bits, splits inside a span are cleared (inner_bits), Whitespace never drops a
// span's bytes (added_bits | inner_bits).  The page summaries keep counting from the DOCUMENT starts.
struct AddedBits { const uint32_t* hard; const uint32_t* inner; const uint32_t* added; };
template <int KIND, bool ADDED = false>
__global__ void __launch_bounds__(K1_THREADS, K1_LEAN_MINBLOCKS)
pretok_lean_kernel(const uint8_t* __restrict__ bytes, int64_t n64, const uint32_t* __restrict__ doc_bits,
                   const uint32_t* __restrict__ cls_tbl, uint32_t* __restrict__ start_bits, uint32_t* __restrict__ drop_bits,
                   uint64_t* __restrict__ page_sum, int n_kb, int kb_per_warp, SwapMasks masks, AddedBits ab = AddedBits{nullptr, nullptr, nullptr}) {
  constexpr unsigned FULL = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31;
  int it_lo, it_hi;
  if (!warp_range(n_kb, kb_per_warp, it_lo, it_hi)) return;
  const uint32_t n = (uint32_t)n64;
  const uint32_t n_chunks = n / CHUNK + 1;
  const At4Global at4{reinterpret_cast<const uint32_t*>(bytes), n};
  const int up = (lane + 31) & 31, down = (lane + 1) & 31;
  const ChunkLoader load{bytes, n, lane};   // load(it, w): it = -1: nothing there

  // carries of my chunk of the previous iteration (lane 31's chunk precedes lane 0's)
  uint32_t kL = 0u, kN = 0u, kS = 0u, kSP = 0u, k_ov = 0u;
  // stage A results of iteration j - 1, waiting for stage B
  uint32_t p_start = 0u, p_drop = 0u, p_lead = 0u, p_head = 0u, p_ds = 0u, p_dsn = 0u, p_s31 = 0u;
  uint32_t p_inner = 0u, p_doc = 0u;              // ADDED only
  PageSummary ps{0u, 0u, 0u};

  uint32_t w[8];
  load(it_lo > 0 ? it_lo - 1 : -1, w);
#pragma unroll 1
  for (int j = it_lo - 1; j <= it_hi; ++j) {
    // ================= stage A: iteration j
    const uint32_t c = (uint32_t)j * 32u + lane, base = c * CHUNK;
    // interior iteration (warp-uniform): this KB and the first chunk of the next one lie inside the batch
    const bool interior = j >= 0 && ((uint32_t)j * 32u + 33u) * CHUNK <= n;
    uint32_t valid = 0xFFFFFFFFu;
    if (!interior) valid = chunk_valid(j >= 0, base, n);
    uint32_t b[8];
    bitslice32(w, b, masks);
    if (j + 1 < it_hi && ((uint32_t)j * 32u + 64u) * CHUNK <= n) {   // prefetch; the common case first: a whole KB inside the batch
      load32(bytes + (uint32_t)(base + 32u * CHUNK), w);          // (j = -1: the sum wraps to lane * 32)
    } else {
      load(j + 1 <= it_hi ? j + 1 : -1, w);      // range / batch ends (the KB after the range is classified too, for its first bytes)
    }
    FastCls m = classify_planes<KIND>(b, valid);
    if (__any_sync(FULL, m.hi != 0u)) {
      if (m.unc) resolve_uncertain(m, at4, base, cls_tbl);
      fill_own(m);
    }
    PrevTop pt;
    pt.L = __shfl_sync(FULL, lane == 31 ? kL : m.L, up);
    pt.S = __shfl_sync(FULL, lane == 31 ? kS : m.S, up);
    if (KIND == PT_GPT2) {
      pt.N = __shfl_sync(FULL, lane == 31 ? kN : m.N, up);
      pt.SP = __shfl_sync(FULL, lane == 31 ? kSP : m.SP, up);
    } else { pt.N = 0u; pt.SP = 0u; }
    if (m.cont & 1u) spill_in(m, pt.L, pt.N, pt.S);
    kL = m.L; kN = m.N; kS = m.S; kSP = m.SP;
    // ds / ds_next: where a new string starts as far as the regex is concerned (ADDED: hard_bits)
    const uint32_t* __restrict__ rbits = ADDED ? ab.hard : doc_bits;
    uint32_t ds, ds_next;
    if (interior) { ds = __ldg(rbits + c); ds_next = __ldg(rbits + c + 1); }
    else { ds = (j >= 0 && c < n_chunks) ? __ldg(rbits + c) : 0u; ds_next = (j >= 0 && c + 1 < n_chunks) ? __ldg(rbits + c + 1) : 0u; }
    uint32_t inner = 0u, keep = 0u, docw = ds;
    if (ADDED && j >= 0 && c < n_chunks) {
      inner = __ldg(ab.inner + c); docw = __ldg(doc_bits + c);
      if (pretok_drops_whitespace(KIND)) keep = inner | __ldg(ab.added + c);
    }
    uint32_t start, drop = 0u;
    if (KIND == PT_GPT2) {
      const FastOut o = fast_gpt2(m, pt, ds, ds_next, base, at4);
      Overflow in; in.bits = __shfl_sync(FULL, lane == 31 ? k_ov : o.ov.bits, up);
      k_ov = o.ov.bits;
      start = apply_overflow(o.start, m.lead, in);
    } else if (KIND == PT_WHITESPACE || KIND == PT_BERT) {
      const FastOut o = KIND == PT_BERT ? fast_bert(m, pt, ds) : fast_whitespace(m, pt, ds);
      start = o.start; drop = o.drop & ~keep;
    } else {
      start = ds & m.lead;
    }
    const uint32_t head = (m.lead & 15u) | ((m.S & 15u) << 4);
    // ================= stage B: iteration j - 1
    if (j > it_lo) {
      const int it = j - 1;
      const uint32_t pc = (uint32_t)it * 32u + lane;
      uint32_t fin = p_start;
      if (KIND == PT_GPT2) {
        const uint32_t xh = __shfl_sync(FULL, lane == 0 ? head : p_head, down);
        fin = finalize_gpt2(fin, p_lead, p_s31, xh & 15u, xh >> 4, p_dsn);
      }
      if (ADDED) fin &= ~p_inner;      // an added token's span is one pre-token
      if (pc < n_chunks) {
        start_bits[pc] = fin;
        if (pretok_drops_whitespace(KIND)) drop_bits[pc] = p_drop;
      }
      ps.add(it, n_kb, n, lane, p_lead, fin & ~p_drop, ADDED ? p_doc : p_ds, page_sum);
    }
    p_start = start; p_drop = drop; p_lead = m.lead; p_head = head; p_ds = ds; p_dsn = ds_next; p_s31 = m.S >> 31;
    if (ADDED) { p_inner = inner; p_doc = docw; }
  }
}

// ---------------------------------------------------------------------------------------------- window form (Llama-3)
// Same streaming structure with the 64-bit window algebra of pretok_logic.cuh (two iterations per trip).  Only
// start_bits is written: the tiktoken pattern removes nothing, every split is kept.

struct DsAtGlobal {
  const uint32_t* __restrict__ doc_bits;
  int64_t n_chunks;
  __device__ __forceinline__ uint32_t operator()(int64_t k) const { return (k >= 0 && k < n_chunks) ? __ldg(doc_bits + k) : 0u; }
};

// The slow path for chunk c, whose window w has a run that reaches its edge.  Out of line, so that the hot loop's
// registers do not change.  llama_carry walks the chunks around c, classified again from global memory.
static __device__ __noinline__ uint32_t llama3_slow_start(Window w, const uint8_t* __restrict__ bytes, uint32_t n, uint32_t c,
                                                          const uint32_t* __restrict__ cls_tbl, const uint32_t* __restrict__ rbits) {
  const uint32_t n_chunks = n / CHUNK + 1;
  const At4Global at4{reinterpret_cast<const uint32_t*>(bytes), n};
  const auto masks = [&](int64_t k) {
    uint32_t wk[8];
    const uint32_t base = (uint32_t)k * CHUNK;
    ChunkLoader{bytes, n, (int)(k & 31)}((int)(k >> 5), wk);   // chunk k = lane k % 32 of iteration k / 32
    return classify_standalone<PT_LLAMA3>(wk, chunk_valid(true, base, n), base, at4, cls_tbl);
  };
  return llama3_slow_path(w, c, n_chunks, masks, DsAtGlobal{rbits, n_chunks}, at4);
}

template <int KIND, bool ADDED = false>
__global__ void __launch_bounds__(K1_THREADS, K1_WINDOW_MINBLOCKS)
pretok_stream_kernel(const uint8_t* __restrict__ bytes, int64_t n64, const uint32_t* __restrict__ doc_bits,
                     const uint32_t* __restrict__ cls_tbl, uint32_t* __restrict__ start_bits,
                     uint64_t* __restrict__ page_sum, int n_kb, int kb_per_warp, AddedBits ab = AddedBits{nullptr, nullptr, nullptr}) {
  static_assert(KIND == PT_LLAMA3, "the window form is the Llama-3 kernel");
  constexpr unsigned FULL = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31;
  int it_lo, it_hi;
  if (!warp_range(n_kb, kb_per_warp, it_lo, it_hi)) return;
  const uint32_t n = (uint32_t)n64;
  const uint32_t n_chunks = n / CHUNK + 1;
  const At4Global at4{reinterpret_cast<const uint32_t*>(bytes), n};
  const int up = (lane + 31) & 31, down = (lane + 1) & 31;

  const ChunkLoader load{bytes, n, lane};   // it = -1: nothing there
  // classes of iteration `it`; `prev` = this lane's classes of the iteration before (lane 31's chunk precedes lane 0's)
  auto classify = [&](const uint32_t w[8], int it, const FastCls& prev, FastCls& m, FastCls& pm) {
    const uint32_t base = ((uint32_t)it * 32u + lane) * CHUNK;
    uint32_t b[8];
    bitslice32(w, b);
    m = classify_planes<KIND>(b, chunk_valid(it >= 0, base, n));
    if (__any_sync(FULL, m.hi != 0u)) {
      if (m.unc) resolve_uncertain(m, at4, base, cls_tbl);
      fill_own(m);
    }
    // the chunk before mine (the window algebra uses the top halves of its class words)
    pm.L = __shfl_sync(FULL, lane == 31 ? prev.L : m.L, up);
    pm.N = __shfl_sync(FULL, lane == 31 ? prev.N : m.N, up);
    pm.S = __shfl_sync(FULL, lane == 31 ? prev.S : m.S, up);
    pm.SP = __shfl_sync(FULL, lane == 31 ? prev.SP : m.SP, up);
    pm.lead = __shfl_sync(FULL, lane == 31 ? prev.lead : m.lead, up);
    pm.NL = __shfl_sync(FULL, lane == 31 ? prev.NL : m.NL, up);
    pm.AP = __shfl_sync(FULL, lane == 31 ? prev.AP : m.AP, up);
    if (m.cont & 1u) spill_in(m, pm.L, pm.N, pm.S);
  };

  PageSummary ps{0u, 0u, 0u};

  // One iteration: classify it+1 (words in w) into nxt / pnxt, refill w with the words of it+3, then boundaries,
  // stores and page summary of iteration `it` (classes in cur / pcur).
  auto step = [&](int it, const FastCls& cur, const FastCls& pcur, FastCls& nxt, FastCls& pnxt, uint32_t w[8]) {
    classify(w, it + 1, cur, nxt, pnxt);
    load(it + 3 <= it_hi ? it + 3 : -1, w);      // prefetch (the KB after the range is classified too, for its first bytes)

    const uint32_t c = (uint32_t)it * 32u + lane, base = c * CHUNK;
    const uint32_t* __restrict__ rbits = ADDED ? ab.hard : doc_bits;   // string starts as the regex sees them
    const uint32_t ds = c < n_chunks ? __ldg(rbits + c) : 0u;
    const uint32_t ds_next = c + 1 < n_chunks ? __ldg(rbits + c + 1) : 0u;
    const uint32_t docw = ADDED ? (c < n_chunks ? __ldg(doc_bits + c) : 0u) : ds;
    uint32_t start;
    {
      // window algebra on [16 B of the previous chunk | mine | 16 B of the next chunk]
      Window wd;
      auto nextw = [&](uint32_t mine, uint32_t theirs) { return __shfl_sync(FULL, lane == 0 ? theirs : mine, down); };
      wd.lead = win(pcur.lead, cur.lead, nextw(cur.lead, nxt.lead)); wd.L = win(pcur.L, cur.L, nextw(cur.L, nxt.L));
      wd.N = win(pcur.N, cur.N, nextw(cur.N, nxt.N)); wd.S = win(pcur.S, cur.S, nextw(cur.S, nxt.S));
      wd.SP = win(pcur.SP, cur.SP, nextw(cur.SP, nxt.SP)); wd.NL = win(pcur.NL, cur.NL, nextw(cur.NL, nxt.NL));
      wd.AP = win(pcur.AP, cur.AP, nextw(cur.AP, nxt.AP));
      const uint32_t ds_prev = (c >= 1u && c - 1u < n_chunks) ? __ldg(rbits + c - 1) : 0u;
      wd.DS = win(ds_prev, ds, ds_next);
      LlamaCarry cy; cy.n_count_before_window = 0; cy.zone_before_window = false; cy.tail_after_window = false;
      const BoundaryOut r = boundaries_llama3(wd, (int64_t)base - 16, at4, cy);
      start = r.start;
      if (r.slow) start = llama3_slow_start(wd, bytes, n, c, cls_tbl, rbits);
    }
    if (ADDED && c < n_chunks) start &= ~__ldg(ab.inner + c);   // an added token's span is one pre-token
    if (c < n_chunks) start_bits[c] = start;
    ps.add(it, n_kb, n, lane, cur.lead, start, docw, page_sum);
  };

  FastCls A, pA, B, pB;   // p*: the chunk before (as far as needed)
  uint32_t w0[8], w1[8];
  {
    FastCls zero;
    zero.lead = zero.cont = zero.hi = zero.L = zero.N = zero.S = zero.SP = zero.AP = zero.NL = zero.unc = 0u;
    load(it_lo - 1, w0);
    classify(w0, it_lo - 1, zero, B, pB);
    load(it_lo, w0);
    classify(w0, it_lo, B, A, pA);
    load(it_lo + 1, w0);
    load(it_lo + 2 <= it_hi ? it_lo + 2 : -1, w1);
  }
  // two iterations per trip, the class registers ping-pong (A holds the even iteration, B the odd one)
  for (int it = it_lo; it < it_hi; it += 2) {
    step(it, A, pA, B, pB, w0);
    if (it + 1 < it_hi) step(it + 1, B, pB, A, pA, w1);
  }
}

}  // namespace b2t
