// model_kernels.cuh -- K2: one tile kernel that turns (bytes, pre-token bitmap) into the token CSR.
//
// Replaces, per 2 KB page of the packed batch (paths relative to tokenizers/src of huggingface/tokenizers):
//   models/bpe/model.rs:465-612 (merge_word, tokenize_with_cache incl. ignore_merges) + models/bpe/word.rs:162-268
//   models/wordpiece/mod.rs:224-283 (greedy longest match, max_input_chars_per_word, [UNK])
//   tokenizer/pre_tokenizer.rs:198-263,329-364 (into_encoding: offsets -> original -> char, word ids)
//   tokenizer/encoding.rs:541-565 (collecting tokens of all splits in order)
//
// Work decomposition: the block owns the pre-tokens that START inside its page (they may run into the halo).
//   * every symbol lives at its byte position in shared memory (id, length, rank of the pair it forms with its right
//     neighbour), so symbols never move: a merge extends the left symbol and zeroes the length of the right one;
//   * every pre-token of up to 24 bytes is first looked up in a per-batch word cache shared by all blocks (the
//     reference caches words too: models/bpe/model.rs:24-90); a hit is a full key compare, so results cannot change;
//   * misses of up to 32 bytes are merged by 8-lane groups, longer ones (up to 256) by a whole warp, pair ranks held in
//     registers: every round the group agrees by shuffles on the leftmost pair of minimal rank (== the reference's
//     heap order (rank, pos) with its stale-entry check) and publishes the result to the cache;
//   * surviving symbol starts are exactly the token starts: a ballot per 32 positions gives the token bitmap, ids /
//     offsets / word ids are written at provisional slots (page's first start + j) and a scan + compaction pass moves
//     them to their final CSR position -- pages never wait for each other.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "b2t_tables.h"
#include "added_kernels.cuh"
#include "long_kernels.cuh"
#include "pretok_logic.cuh"

namespace b2t {

constexpr int TILE = PAGE;
constexpr int MODEL_THREADS = 256;
constexpr int THREAD_PATH_MAX = 32;  // pre-tokens up to this many bytes are merged by an 8-lane group, longer ones by a warp
enum { MODEL_BPE = 0, MODEL_WORDPIECE = 1 };
enum { F_OFFSETS = 1u, F_WORD_IDS = 2u, F_BYTE_OFFSETS = 4u };
constexpr int MAX_LONG_PER_PAGE = TILE / (LONG_PRETOK_MIN + 1) + 1;  // 8

struct ModelParams {
  const uint8_t* bytes; int64_t n;
  const uint32_t* start_bits; const uint32_t* drop_bits; const uint32_t* doc_bits;
  // BPE: exact cuts inside long pre-tokens (long_kernels.cuh soft_cut) and the pages that hold any; the page kernel merges
  // the pieces like pre-tokens of their own, word ids and offsets keep following start_bits
  const uint32_t* soft_bits; const uint8_t* page_soft;
  const uint64_t* page_carry; const uint64_t* block_carry; const uint32_t* page_first_doc;
  const uint64_t* doc_off; uint32_t n_docs;
  uint32_t flags;
  uint32_t* ids; uint32_t* offsets; uint32_t* word_ids; uint64_t* row_ptr;
  // pass 1 writes the tokens of page t at the provisional slots [tile_first[t], tile_first[t] + tile_count[t]) of ids / offsets /
  // word_ids (first pre-token start of the page: a page never has more tokens than bytes up to the next page's first start),
  // row_ptr holds page-local token counts; tile_scan + compact_kernel + row_ptr_fix_kernel then produce the final CSR.
  uint32_t* tile_count; uint32_t* tile_first; uint32_t* err_flag;
  int64_t n_tiles;
  // long BPE pre-tokens resolved by the pre-pass (long_kernels.cuh)
  const int32_t* page_long; const LongDesc* long_desc; const uint4* long_out;
  // per-batch word cache (cleared at the start of every batch): pre-token bytes -> its token list
  uint4* wcache; uint32_t wcache_mask; int wcache_on;   // wcache_on = 0: every pre-token is merged (the reference's cache_capacity(0))
  // ByteLevel add_prefix_space: bit p set <=> byte p of the (re-packed) batch is an inserted prefix space (else NULL)
  const uint32_t* prefix_bits;
  // added-token extraction (added_kernels.cuh): bit p <=> an added token's span starts at byte p, its id is in the list of
  // the page; NULL when the batch did not go through the extraction.  flag_added: mark those tokens with bit 31 of the id.
  const uint32_t* added_bits; const uint32_t* added_head; const uint2* added_pool; uint32_t flag_added;
  DeviceTables t;
};

__device__ __forceinline__ uint64_t merge_lookup(const DeviceTables& t, uint32_t a, uint32_t b) {
  const uint32_t hf = pair_hash(a, b);
  uint32_t h = hf & t.merge_mask;
  while (true) {
    uint4 e = __ldg(t.merge_tbl + h);
    if (e.x == a && e.y == b) return ((uint64_t)e.z << 32) | e.w;
    if (e.x == EMPTY_KEY) return NO_MERGE;
    h = (h + 1) & t.merge_mask;
  }
}

// exclusive prefix of popcounts over nw (<= 96) words, by one full warp; returns the total
__device__ __forceinline__ int warp_prefix_words(const uint32_t* bits, uint16_t* pref, int nw, int lane) {
  int c0 = 0, c1 = 0, c2 = 0;
  int i = lane * 3;
  if (i < nw) c0 = __popc(bits[i]);
  if (i + 1 < nw) c1 = __popc(bits[i + 1]);
  if (i + 2 < nw) c2 = __popc(bits[i + 2]);
  int tot = c0 + c1 + c2, inc = tot;
#pragma unroll
  for (int s = 1; s < 32; s <<= 1) {
    int o = __shfl_up_sync(0xFFFFFFFFu, inc, s);
    if (lane >= s) inc += o;
  }
  int ex = inc - tot;
  if (i < nw) pref[i] = (uint16_t)ex;
  if (i + 1 < nw) pref[i + 1] = (uint16_t)(ex + c0);
  if (i + 2 < nw) pref[i + 2] = (uint16_t)(ex + c0 + c1);
  return __shfl_sync(0xFFFFFFFFu, inc, 31);
}

__device__ __forceinline__ uint32_t mask_le(int b) { return b >= 31 ? 0xFFFFFFFFu : ((2u << b) - 1u); }

// One word per byte position of the page: token id (low 20 bits) and token length in bytes (high 12 bits); length 0 =
// no token starts here.  (Ids and lengths used to be two arrays; one array leaves 4.5 KB of the SM's shared memory /
// L1 pool to L1, where the merge-table probes of the merge rounds then hit.)  b2t_engine_create refuses ids >= 2^20.
constexpr int TOK_ID_BITS = 20;
__device__ __forceinline__ uint32_t tok_pack(uint32_t id, int len) { return id | ((uint32_t)len << TOK_ID_BITS); }
__device__ __forceinline__ int tok_len(uint32_t x) { return (int)(x >> TOK_ID_BITS); }
__device__ __forceinline__ uint32_t tok_id(uint32_t x) { return x & ((1u << TOK_ID_BITS) - 1u); }


// ------------------------------------------------------------------------------------------------ word cache
// The reference keeps a per-thread word cache in front of merge_word (models/bpe/model.rs:24-90, 568-586) because
// natural text repeats its words; it has no semantic effect.  Same idea here, per batch and shared by all blocks: a
// pre-token of up to 24 bytes whose result has up to 6 tokens is published once and reused by every later occurrence
// in the batch (full key comparison, so a hit is exact).  Slot = 64 bytes:
//   q0 = {tag lo, tag hi, key[0], key[1]}   q1 = {key[2..5]}   q2 = {ntok | len0..2, len3..5 | -, id0, id1}   q3 = {id2..id5}
// tag: 0 = free, BUSY | fp = being written, READY | fp = valid.  Writers publish with payload -> fence -> tag.
constexpr int WC_MAX_BYTES = 24, WC_MAX_TOK = 6, WC_PROBES = 4;
// Cache misses of up to P4_SPLIT_BYTES bytes are merged by 8 lanes x 2 positions, longer ones (<= THREAD_PATH_MAX) by
// 8 lanes x 4, in separate passes: the groups of a warp step through their merge rounds together, so a warp should
// hold words of similar length.  Fewer lanes per short word mean more words per warp and so more rounds per pass: the
// rounds are L2-latency bound, not lane bound.
constexpr int P4_SPLIT_BYTES = 16;
constexpr int P4_SHORT_G = 8;
template <int V> struct IntTag { static constexpr int value = V; };
#define B2T_WC_READY (1ull << 63)
#define B2T_WC_BUSY (1ull << 62)
#define B2T_WC_FP ((1ull << 62) - 1ull)

struct WordKey {
  uint32_t k[6];
  uint32_t slot;
  unsigned long long fp;
};

// 24 zero-padded bytes of the pre-token [s, s + len) from shared memory + their hash
__device__ __forceinline__ void wc_make_key(const uint8_t* s_byte, int s, int len, WordKey& key) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(s_byte) + (s >> 2);
  const uint32_t sh = (uint32_t)(s & 3) * 8u;
  uint32_t a0 = w[0], a1 = w[1], a2 = w[2], a3 = w[3], a4 = w[4], a5 = w[5], a6 = w[6];
  uint32_t k[6] = {__funnelshift_r(a0, a1, sh), __funnelshift_r(a1, a2, sh), __funnelshift_r(a2, a3, sh),
                   __funnelshift_r(a3, a4, sh), __funnelshift_r(a4, a5, sh), __funnelshift_r(a5, a6, sh)};
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    // bytes of word i that belong to the pre-token: v = clamp(len - 4 i, 0, 4); mask = the low 8 v bits, as one clamped
    // funnel shift (a shift count above 32 counts as 32 and yields 0; v <= 0 gives a count >= 32)
    const int v = min(len - 4 * i, 4);
    const uint32_t m = __funnelshift_rc(0xFFFFFFFFu, 0u, (uint32_t)(32 - 8 * v));
    key.k[i] = k[i] & m;
  }
  uint32_t a = key.k[0] ^ (key.k[2] * 0x9E3779B1u) ^ (key.k[4] * 0x85EBCA77u);
  uint32_t b = key.k[1] ^ (key.k[3] * 0xC2B2AE3Du) ^ (key.k[5] * 0x27D4EB2Fu);
  a = (a ^ (uint32_t)len) * 0x2C1B3C6Du; b = (b + a) * 0x297A2D39u;
  a ^= b >> 15; a *= 0x85EBCA6Bu; b ^= a >> 13; b *= 0xC2B2AE35u; a ^= b >> 16;
  key.slot = a;
  key.fp = ((((unsigned long long)b << 32) | a) ^ ((unsigned long long)len << 56)) & B2T_WC_FP;
  if (key.fp == 0) key.fp = 1;
}

// Memory-model note.  A slot is written once per batch (the table is zeroed, stream-ordered, before the kernel) and never
// changes after that, readers take no lock and no fence -- an acquire load costs an L1 invalidation (CCTL.IVALL) per
// probe on this architecture, and the merge-table probes live in L1.  Instead every 32-bit word of a written slot is
// NON-ZERO by construction (key words and ids are stored complemented: a key word of 0xFFFFFFFF cannot occur in UTF-8,
// ids are < 2^20; the two length words carry a marker bit), all accesses are strong (.relaxed.gpu, single-copy atomic
// per 32-bit word), and a reader accepts a slot only if the words it uses are non-zero and the whole key matches.  A word
// that is not yet visible reads as zero, which is a miss: the pre-token is merged, the result is the same.
__device__ __forceinline__ uint4 ld_relaxed_v4(const uint4* p) {
  uint4 v;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_v4(uint4* p, uint4 v) {
  asm volatile("st.relaxed.gpu.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
constexpr uint32_t WC_LEN_MARK = 0x80000000u;   // bit 31 of the second length word: always set in a written slot

// Returns true on a hit (tokens written to s_tok).
__device__ __forceinline__ bool wc_lookup(uint4* cache, uint32_t mask, const WordKey& key, int s, uint32_t* s_tok) {
  uint32_t slot = key.slot & mask;
#pragma unroll 1
  for (int pr = 0; pr < WC_PROBES; ++pr, slot = (slot + 1) & mask) {
    const uint4* q = cache + (size_t)slot * 4;
    const uint4 q0 = ld_relaxed_v4(q);
    const unsigned long long tag = ((unsigned long long)q0.y << 32) | q0.x;
    if (tag == 0ull) return false;
    if (tag != (B2T_WC_READY | key.fp)) {
      if (tag == (B2T_WC_BUSY | key.fp)) return false;  // someone is publishing this very word: just compute it
      continue;
    }
    if (q0.z != ~key.k[0] || q0.w != ~key.k[1]) continue;
    const uint4 q1 = ld_relaxed_v4(q + 1);
    if (q1.x != ~key.k[2] || q1.y != ~key.k[3] || q1.z != ~key.k[4] || q1.w != ~key.k[5]) continue;
    const uint4 q2 = ld_relaxed_v4(q + 2), q3 = ld_relaxed_v4(q + 3);
    const int ntok = (int)(q2.x & 0xFFu);
    const uint32_t cids[6] = {q2.z, q2.w, q3.x, q3.y, q3.z, q3.w};   // complemented ids
    const uint32_t lens[6] = {(q2.x >> 8) & 0xFFu, (q2.x >> 16) & 0xFFu, q2.x >> 24, q2.y & 0xFFu, (q2.y >> 8) & 0xFFu, (q2.y >> 16) & 0xFFu};
    bool ok = ntok != 0 && (q2.y & WC_LEN_MARK);
#pragma unroll
    for (int t = 0; t < WC_MAX_TOK; ++t) ok = ok && (t >= ntok || cids[t] != 0u);
    if (!ok) return false;   // part of the slot is not visible yet: a miss
    int pos = s;
#pragma unroll
    for (int t = 0; t < WC_MAX_TOK; ++t)
      if (t < ntok) { s_tok[pos] = tok_pack(~cids[t], (int)lens[t]); pos += (int)lens[t]; }
    return true;
  }
  return false;
}

// Publish the merged pre-token [s, e) (symbols chained by their lengths) into the first free slot of its probe sequence.
__device__ __forceinline__ void wc_publish(uint4* cache, uint32_t mask, const WordKey& key, int s, int e, const uint32_t* s_tok) {
  uint32_t ids[6] = {0, 0, 0, 0, 0, 0}, lens[6] = {0, 0, 0, 0, 0, 0};
  int nt = 0, p = s;
  while (p < e) {
    if (nt == WC_MAX_TOK) return;  // too many tokens for a slot
    const uint32_t tk = s_tok[p];
    const int l = tok_len(tk);
#pragma unroll
    for (int t = 0; t < WC_MAX_TOK; ++t) if (t == nt) { ids[t] = tok_id(tk); lens[t] = (uint32_t)l; }
    ++nt; p += l;
  }
  uint32_t slot = key.slot & mask;
#pragma unroll 1
  for (int pr = 0; pr < WC_PROBES; ++pr, slot = (slot + 1) & mask) {
    uint4* q = cache + (size_t)slot * 4;
    unsigned long long* tagp = reinterpret_cast<unsigned long long*>(q);
    unsigned long long tag = *reinterpret_cast<volatile unsigned long long*>(tagp);
    if (tag == 0ull) tag = atomicCAS(tagp, 0ull, B2T_WC_BUSY | key.fp);
    if (tag == 0ull) {  // the slot is ours
      uint32_t* kw = reinterpret_cast<uint32_t*>(q);
      asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1, %2};" ::"l"(kw + 2), "r"(~key.k[0]), "r"(~key.k[1]) : "memory");
      st_relaxed_v4(q + 1, make_uint4(~key.k[2], ~key.k[3], ~key.k[4], ~key.k[5]));
      st_relaxed_v4(q + 2, make_uint4((uint32_t)nt | (lens[0] << 8) | (lens[1] << 16) | (lens[2] << 24), lens[3] | (lens[4] << 8) | (lens[5] << 16) | WC_LEN_MARK, ~ids[0], ~ids[1]));
      st_relaxed_v4(q + 3, make_uint4(~ids[2], ~ids[3], ~ids[4], ~ids[5]));
      __threadfence();                                  // not needed for correctness (see above); it makes the slot usable sooner
      atomicExch(tagp, B2T_WC_READY | key.fp);
      return;
    }
    if ((tag & B2T_WC_FP) == key.fp) return;  // (probably) the same word, already there or on its way
  }
}

// models/bpe/model.rs:558-567 (ignore_merges): is the whole pre-token a vocabulary entry?  Writes it (one token) to s_tok[s].
__device__ __forceinline__ bool vocab_whole_word(const DeviceTables& t, const uint8_t* s_byte, int s, int len, uint32_t* s_tok) {
  StrHash h; strhash_init(h);
  for (int p = s; p < s + len; ++p) strhash_byte(h, s_byte[p]);
  strhash_fin(h);
  uint32_t slot = h.h1 & t.word_mask;
  while (true) {
    const uint4 en = __ldg(t.word_tbl + slot);
    if (en.z == EMPTY_KEY) return false;
    if (en.x == h.h2 && en.y == (uint32_t)len) {
      const uint8_t* q = t.word_pool + en.w;
      bool same = true;
      for (int i = 0; i < len; ++i) if (__ldg(q + i) != s_byte[s + i]) { same = false; break; }
      if (same) { s_tok[s] = tok_pack(en.z, len); return true; }
    }
    slot = (slot + 1) & t.word_mask;
  }
}

// ------------------------------------------------------------------------------------------------ cooperative merge
// G lanes resolve one pre-token [s, e) of up to G * J bytes: lane g owns the positions s + g + G * j (j < J) and
// keeps the rank / new id of the pair that starts at each of them in registers.  Every round the group agrees on
// the leftmost pair of minimal rank (== the reference's heap order (rank, pos), models/bpe/word.rs:28-35), its owner
// merges, and the (at most two) pairs that changed are looked up again.  All groups of a warp step together; the
// control flow is warp-uniform, so nothing diverges -- idle groups are predicated off.
template <int G, int J>
__device__ __forceinline__ void coop_bpe(const DeviceTables& t, const uint8_t* s_byte, uint32_t* s_tok, int s, int e,
                                         bool active, int gl) {
  uint32_t rk[J], ni[J];
#pragma unroll
  for (int j = 0; j < J; ++j) {
    const int p = s + gl + G * j;
    rk[j] = 0xFFFFFFFFu; ni[j] = 0u;
    if (active && p < e) s_tok[p] = tok_pack(__ldg(t.byte_to_id + s_byte[p]), 1);
  }
  __syncwarp();
#pragma unroll
  for (int j = 0; j < J; ++j) {
    const int p = s + gl + G * j;
    if (active && p + 1 < e) { const uint64_t v = merge_lookup(t, tok_id(s_tok[p]), tok_id(s_tok[p + 1])); rk[j] = (uint32_t)(v >> 32); ni[j] = (uint32_t)v; }
  }
  while (true) {
    // leftmost minimum over my positions (they grow with j), then over the group
    uint32_t br = 0xFFFFFFFFu, bpos = 0x7FFFFFFFu;
#pragma unroll
    for (int j = 0; j < J; ++j) if (rk[j] < br) { br = rk[j]; bpos = (uint32_t)(s + gl + G * j); }
#pragma unroll
    for (int st = G / 2; st >= 1; st >>= 1) {
      const uint32_t orr = __shfl_xor_sync(0xFFFFFFFFu, br, st), op = __shfl_xor_sync(0xFFFFFFFFu, bpos, st);
      if (orr < br || (orr == br && op < bpos)) { br = orr; bpos = op; }
    }
    const bool have = active && br != 0xFFFFFFFFu;
    if (!__any_sync(0xFFFFFFFFu, have)) break;
    const int bp = (int)bpos;
    int nx = 0, pv = -1;
    uint32_t nid = 0;
    if (have) {
      // everybody in the group derives the same facts from shared memory (read before the owner writes)
      const int ql = tok_len(s_tok[bp]);
      const int q = bp + ql;
      nx = q + tok_len(s_tok[q]);
      pv = bp - 1;
      while (pv >= s && tok_len(s_tok[pv]) == 0) --pv;
    }
    __syncwarp();
    if (have) {
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int p = s + gl + G * j;
        if (p == bp) {  // owner of the winning pair: merge right into left
          nid = ni[j];
          const int q = bp + tok_len(s_tok[bp]);
          s_tok[bp] = tok_pack(nid, nx - bp); s_tok[q] = 0u;
        }
        if (p > bp && p < nx) rk[j] = 0xFFFFFFFFu;  // the swallowed symbol no longer starts a pair
      }
    }
    __syncwarp();
    if (have) {
      const uint32_t newid = tok_id(s_tok[bp]);
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int p = s + gl + G * j;
        if (p == bp) {
          rk[j] = 0xFFFFFFFFu;
          if (nx < e) { const uint64_t v = merge_lookup(t, newid, tok_id(s_tok[nx])); rk[j] = (uint32_t)(v >> 32); ni[j] = (uint32_t)v; }
        } else if (p == pv) {
          const uint64_t v = merge_lookup(t, tok_id(s_tok[pv]), newid); rk[j] = (uint32_t)(v >> 32); ni[j] = (uint32_t)v;
        }
      }
    }
  }
}


#ifndef B2T_MINBLOCKS
#define B2T_MINBLOCKS 8  // 8 blocks/SM (32 regs, small spills) rather than 5 (48 regs): the kernel is latency-bound
#endif
template <int MODEL>
__global__ void __launch_bounds__(MODEL_THREADS, B2T_MINBLOCKS) model_tile_kernel(const ModelParams P) {
  constexpr int HALO = MODEL == MODEL_BPE ? 256 : 416;
  constexpr int SPAN = TILE + HALO;
  constexpr int NW = SPAN / 32;
  constexpr int TW = TILE / 32;
  static_assert(NW <= 96, "warp_prefix_words handles <= 96 words");
  __shared__ __align__(16) uint8_t s_byte[SPAN];
  __shared__ __align__(16) uint32_t s_tok[SPAN];   // tok_pack(id, length) of the token that starts at each position
  __shared__ uint32_t s_startb[NW + 1], s_keptb[NW + 1], s_leadb[NW + 1], s_tokb[NW + 1], s_dsb[TW + 1], s_addedb[TW + 1];
  __shared__ uint16_t s_apref[NW + 1], s_spref[NW + 1], s_lpref[NW + 1], s_tpref[NW + 1];
  __shared__ int16_t s_dlast[TW + 1];
  __shared__ uint16_t s_pt[TILE + 2];
  __shared__ uint16_t s_mq[TILE / THREAD_PATH_MAX + 2];
  __shared__ uint16_t s_list[SPAN];  // P3/P4: pre-tokens the word cache did not resolve; P7: positions of the tokens
  uint16_t* const s_miss = s_list;
  uint16_t* const s_tokpos = s_list;
  __shared__ int s_nmiss, s_nmiss_hi;  // misses queued from the front (short) and from the back (longer) of s_miss
  __shared__ int s_tile, s_next, s_nmq, s_P, s_Elast, s_long, s_ntok, s_ntot, s_anysoft;
  __shared__ unsigned long long s_excl;
  __shared__ long long s_long_end, s_span_doc_start;
  __shared__ int s_long_chars;
  __shared__ int s_nl;                                   // long BPE pre-tokens that start in this page
  __shared__ uint16_t s_lk[MAX_LONG_PER_PAGE + 1];       // their pre-token indices, in position order
  __shared__ int s_lcum[MAX_LONG_PER_PAGE + 2];          // exclusive prefix of their token counts
  __shared__ unsigned long long s_loff[MAX_LONG_PER_PAGE + 1];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NWARPS = MODEL_THREADS / 32;
  if (tid == 0) {
    s_tile = (int)blockIdx.x;
    s_next = 0; s_nmq = 0; s_long = 0; s_long_chars = 0; s_nl = 0; s_nmiss = 0; s_nmiss_hi = 0; s_anysoft = 0; s_lcum[0] = 0;
  }
  __syncthreads();
  const int64_t t = s_tile;
  if (t >= P.n_tiles) return;
  const int64_t base = t * TILE;
  const int64_t n = P.n;
  const int64_t n_chunks = n / CHUNK + 1;

  // ---------------------------------------------------------------- P0: stage bytes and bitmaps
  for (int i = tid; i < SPAN / 16; i += MODEL_THREADS) {
    int64_t g = base + (int64_t)i * 16;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (g + 16 <= n) v = __ldg(reinterpret_cast<const uint4*>(P.bytes + g));
    else if (g < n) {
      uint32_t w[4] = {0, 0, 0, 0};
      for (int k = 0; k < 16 && g + k < n; ++k) w[k >> 2] |= (uint32_t)__ldg(P.bytes + g + k) << (8 * (k & 3));
      v = make_uint4(w[0], w[1], w[2], w[3]);
    }
    reinterpret_cast<uint4*>(s_byte)[i] = v;
  }
  for (int w = tid; w <= NW; w += MODEL_THREADS) {
    int64_t gw = base / 32 + w;
    uint32_t sb = (w < NW && gw < n_chunks) ? __ldg(P.start_bits + gw) : 0u;
    uint32_t db = (MODEL == MODEL_WORDPIECE && w < NW && gw < n_chunks) ? __ldg(P.drop_bits + gw) : 0u;
    uint32_t sf = 0u;
    if (MODEL == MODEL_BPE && w < NW && gw < n_chunks && __ldg(P.page_soft + (gw >> 6))) { sf = __ldg(P.soft_bits + gw); if (sf) s_anysoft = 1; }
    s_startb[w] = sb | sf;   // where a unit of merging starts: splits of the pre-tokenizer + exact cuts of long ones
    s_keptb[w] = sb & ~db;   // splits of the pre-tokenizer that the reference keeps (word ids)
    if (w <= TW) s_dsb[w] = (w < TW && gw < n_chunks) ? __ldg(P.doc_bits + gw) : 0u;
    if (w <= TW) s_addedb[w] = (P.added_bits && w < TW && gw < n_chunks) ? __ldg(P.added_bits + gw) : 0u;
  }
  __syncthreads();
  // lead bits (16 bytes per thread: continuation-byte flags by SWAR, two threads make one bitmap word) + symbol init
  static_assert(SPAN / 16 <= MODEL_THREADS && (SPAN / 16) % 2 == 0, "one pass, thread pairs inside a warp");
  {
    const int i = tid;
    const bool act = i < SPAN / 16;
    const uint4 v = act ? reinterpret_cast<const uint4*>(s_byte)[i] : make_uint4(0u, 0u, 0u, 0u);
    const uint32_t c0 = v.x & ~(v.x << 1) & 0x80808080u, c1 = v.y & ~(v.y << 1) & 0x80808080u,
                   c2 = v.z & ~(v.z << 1) & 0x80808080u, c3 = v.w & ~(v.w << 1) & 0x80808080u;   // 10xxxxxx
    const uint32_t cont = movemask2(c0, c1) | (movemask2(c2, c3) << 8);
    const int64_t lim = n - base - (int64_t)i * 16;          // valid bytes from this thread's first position on
    const uint32_t valid = lim >= 16 ? 0xFFFFu : (lim <= 0 ? 0u : ((1u << (int)lim) - 1u));
    const uint32_t lead16 = ~cont & valid;
    const uint32_t other = __shfl_down_sync(0xFFFFFFFFu, lead16, 1);
    if (act && !(i & 1)) s_leadb[i >> 1] = lead16 | (other << 16);
    if (act) {   // token starts are written by whoever resolves the pre-token
      uint4* z = reinterpret_cast<uint4*>(s_tok) + 4 * i;
      z[0] = make_uint4(0u, 0u, 0u, 0u); z[1] = make_uint4(0u, 0u, 0u, 0u); z[2] = make_uint4(0u, 0u, 0u, 0u); z[3] = make_uint4(0u, 0u, 0u, 0u);
    }
  }
  if (tid == 0) s_leadb[NW] = 0u;
  __syncthreads();

  // ---------------------------------------------------------------- P1/P2: prefixes, end of the last pre-token
  if (warp == 0) {
    int tot = warp_prefix_words(s_startb, s_apref, TW, lane);  // all starts inside the page
    if (lane == 0) s_P = tot;
  } else if (warp == 1) {
    warp_prefix_words(s_keptb, s_spref, NW, lane);
  } else if (warp == 2) {
    warp_prefix_words(s_leadb, s_lpref, NW, lane);
  } else if (warp == 3) {
    // first start bit at a position >= TILE (the end of the page's last pre-token)
    int found = SPAN;
    for (int w = TW + lane; w < NW; w += 32) {
      uint32_t b = s_startb[w];
      if (b) { found = w * 32 + (__ffs((int)b) - 1); break; }
    }
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) found = min(found, __shfl_xor_sync(0xFFFFFFFFu, found, s));
    int64_t lim = n - base;  // bytes available from the page start
    int is_long = 0;
    long long long_end = 0;
    if (found >= SPAN) {
      if (lim <= SPAN) found = (int)lim;
      else {
        // no start inside the halo: the last pre-token is LONG.  Find its true end in the global bitmap.
        is_long = 1;
        int64_t gw = (base + SPAN) / 32;
        long long e = (MODEL == MODEL_BPE) ? n : -1;  // BPE: the pre-pass already knows the end
        while (e < 0) {
          int64_t w = gw + lane;
          uint32_t b = (w < n_chunks) ? __ldg(P.start_bits + w) : 0u;
          uint32_t any = __ballot_sync(0xFFFFFFFFu, b != 0u);
          if (any) {
            int l = __ffs((int)any) - 1;
            uint32_t bb = __shfl_sync(0xFFFFFFFFu, b, l);
            e = (gw + l) * 32 + (__ffs((int)bb) - 1);
          } else if (gw + 32 >= n_chunks) e = n;
          gw += 32;
        }
        long_end = e < n ? e : n;
        found = SPAN;
      }
    } else if (found > lim) found = (int)lim;
    if (lane == 0) { s_Elast = found; s_long = is_long; s_long_end = long_end; }
  } else if (warp == 4) {
    // last doc start strictly before each word of the page
    int mine0 = -1, mine1 = -1;  // lane handles words 2*lane, 2*lane+1
    uint32_t b0 = s_dsb[2 * lane], b1 = s_dsb[2 * lane + 1];
    int last0 = b0 ? (2 * lane) * 32 + 31 - __clz((int)b0) : -1;
    int last1 = b1 ? (2 * lane + 1) * 32 + 31 - __clz((int)b1) : -1;
    int mx = max(last0, last1), inc = mx;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      int o = __shfl_up_sync(0xFFFFFFFFu, inc, s);
      if (lane >= s) inc = max(inc, o);
    }
    int before = __shfl_up_sync(0xFFFFFFFFu, inc, 1);
    if (lane == 0) before = -1;
    mine0 = before; mine1 = max(before, last0);
    s_dlast[2 * lane] = (int16_t)mine0; s_dlast[2 * lane + 1] = (int16_t)mine1;
    if (lane == 31) s_dlast[TW] = (int16_t)inc;
  } else if (warp == 5 && lane == 0) {
    // byte position of the start of the document that spans into this page (for byte offsets)
    uint32_t fd = __ldg(P.page_first_doc + t);
    s_span_doc_start = fd > 0 ? (long long)__ldg(P.doc_off + fd - 1) : 0;
  }
  __syncthreads();
  const int Pn = s_P;
  const int Elast = s_Elast;
  const int is_long = s_long && Pn > 0;  // without a start in the page the long pre-token belongs to an earlier page
  if (tid < TW) {
    uint32_t bits = s_startb[tid];
    int idx = s_apref[tid];
    while (bits) { s_pt[idx++] = (uint16_t)(tid * 32 + __ffs((int)bits) - 1); bits &= bits - 1u; }
  }
  if (tid == 0) s_pt[Pn] = (uint16_t)Elast;
  __syncthreads();
  const int first = Pn ? (int)s_pt[0] : Elast;
  // WordPiece: a split that does not fit the halo is [UNK] (handled below).  BPE: pre-tokens longer than LONG_PRETOK_MIN were
  // resolved by the pre-pass; collect them (position order) and blank their bytes so the page logic skips them.
  const int Eproc = Pn ? ((MODEL == MODEL_WORDPIECE && is_long) ? (int)s_pt[Pn - 1] : Elast) : 0;
  const int Pproc = (MODEL == MODEL_WORDPIECE && is_long) ? Pn - 1 : Pn;
  if (MODEL == MODEL_BPE) {
    int any_long = 0;
    for (int k = tid; k < Pn; k += MODEL_THREADS)
      if ((int)s_pt[k + 1] - (int)s_pt[k] > LONG_PRETOK_MIN) { int i = atomicAdd(&s_nl, 1); if (i < MAX_LONG_PER_PAGE) s_lk[i] = (uint16_t)k; any_long = 1; }
    if (__syncthreads_or(any_long)) {   // (almost every page: no long pre-token, one barrier instead of three)
    if (tid == 0) {
      int nl = s_nl;
      if (nl > MAX_LONG_PER_PAGE) { nl = MAX_LONG_PER_PAGE; atomicOr(P.err_flag, ERR_INTERNAL); }
      for (int a = 1; a < nl; ++a) { uint16_t v = s_lk[a]; int b = a - 1; while (b >= 0 && s_lk[b] > v) { s_lk[b + 1] = s_lk[b]; --b; } s_lk[b + 1] = v; }
      const int32_t slot0 = nl ? __ldg(P.page_long + t) : 0;
      if (nl && slot0 < 0) { atomicOr(P.err_flag, ERR_INTERNAL); nl = 0; }
      int cum = 0;
      for (int a = 0; a < nl; ++a) {
        const LongDesc d = P.long_desc[slot0 + a];
        if (d.start != base + s_pt[s_lk[a]]) atomicOr(P.err_flag, ERR_INTERNAL);
        s_lcum[a] = cum; s_loff[a] = d.pool_off;
        cum += (d.pool_off == ~0ull) ? 0 : (int)d.ntok;
      }
      s_lcum[nl] = cum;
      s_nl = nl;
    }
    __syncthreads();
    for (int a = 0; a < s_nl; ++a) {
      const int ls = s_pt[s_lk[a]], le = min((int)s_pt[s_lk[a] + 1], SPAN);
      for (int pos = ls + tid; pos < le; pos += MODEL_THREADS) s_tok[pos] = 0u;
    }
    __syncthreads();
    }
  }
  const int n_longs = MODEL == MODEL_BPE ? s_nl : 0;
  // [s, e) is a piece of a cut pre-token (not a whole split of the pre-tokenizer): with ignore_merges the whole-word rule
  // and the word cache (whose entries follow that rule) do not apply to it
  const bool any_soft = MODEL == MODEL_BPE && s_anysoft != 0;
  auto is_piece = [&](int s, int e) -> bool {
    if (!any_soft) return false;
    const bool real_s = (s_keptb[s >> 5] >> (s & 31)) & 1u;
    const bool real_e = base + e >= n || (e < SPAN && ((s_keptb[e >> 5] >> (e & 31)) & 1u));
    return !(real_s && real_e);
  };
  // number of long-path tokens that precede page position x
  auto long_tokens_before = [&](int x) -> int {
    int c = 0;
    for (int a = 0; a < n_longs; ++a) if ((int)s_pt[s_lk[a]] < x) c = s_lcum[a + 1];
    return c;
  };

  // the pre-token that starts at s (inside the page) is an added token's span: its id comes from the page's list
  auto added_at = [&](int s) -> bool { return P.added_bits != nullptr && ((s_addedb[s >> 5] >> (s & 31)) & 1u); };
  auto added_id = [&](int s) -> uint32_t {
    for (uint32_t i = __ldg(P.added_head + t); i != ADDED_NIL;) {
      const uint2 v = __ldg(P.added_pool + i);
      if ((int)(v.x & (uint32_t)(PAGE - 1)) == s) return v.x >> 11;
      i = v.y;
    }
    atomicOr(P.err_flag, ERR_INTERNAL);
    return 0u;
  };
  if (MODEL == MODEL_BPE) {
    // -------------------------------------------------------------- P3: word cache, one pre-token per thread
    // (static assignment: a lookup costs the same for every lane, so the warp stays converged)
    for (int k0 = 0; k0 < Pproc; k0 += MODEL_THREADS) {
      const int k = k0 + tid;
      int kind = 0;  // 0 = resolved / nothing to do, 1 = miss (<= 32 bytes), 2 = medium (33..256 bytes)
      if (k < Pproc) {
        const int s = s_pt[k], e = s_pt[k + 1], len = e - s;
        if (added_at(s)) { s_tok[s] = tok_pack(added_id(s), len); kind = 0; }   // an added token: one token, whatever the model says
        else if (len > LONG_PRETOK_MIN) kind = 0;  // resolved by the pre-pass
        else if (len > THREAD_PATH_MAX) kind = 2;
        else {
          bool hit = false;
          if (P.wcache_on && len <= WC_MAX_BYTES && !(P.t.ignore_merges && is_piece(s, e))) {
            WordKey key;
            wc_make_key(s_byte, s, len, key);
            hit = wc_lookup(P.wcache, P.wcache_mask, key, s, s_tok);
          }
          kind = hit ? 0 : 1;
        }
      }
      // warp-aggregated queue appends
      // the four groups of a warp step through their merges together, so pre-tokens of similar length should share a
      // warp: short misses queue from the front of s_miss, longer ones from the back
      const bool longer = kind == 1 && (int)s_pt[k + 1] - (int)s_pt[k] > P4_SPLIT_BYTES;
      const unsigned mm = __ballot_sync(0xFFFFFFFFu, kind == 1 && !longer), mh = __ballot_sync(0xFFFFFFFFu, longer),
                     mq = __ballot_sync(0xFFFFFFFFu, kind == 2);
      int bm = 0, bh = 0, bq = 0;
      if (lane == 0) {
        if (mm) bm = atomicAdd(&s_nmiss, __popc(mm));
        if (mh) bh = atomicAdd(&s_nmiss_hi, __popc(mh));
        if (mq) bq = atomicAdd(&s_nmq, __popc(mq));
      }
      bm = __shfl_sync(0xFFFFFFFFu, bm, 0); bh = __shfl_sync(0xFFFFFFFFu, bh, 0); bq = __shfl_sync(0xFFFFFFFFu, bq, 0);
      if (kind == 1 && !longer) s_miss[bm + __popc(mm & ((1u << lane) - 1u))] = (uint16_t)k;
      if (longer) s_miss[SPAN - 1 - (bh + __popc(mh & ((1u << lane) - 1u)))] = (uint16_t)k;
      if (kind == 2) s_mq[bq + __popc(mq & ((1u << lane) - 1u))] = (uint16_t)k;
    }
    __syncthreads();
    // -------------------------------------------------------------- P4a: misses, G lanes per pre-token (<= 32 bytes)
    {
      const int n_short = s_nmiss, n_longer = s_nmiss_hi;
      // G lanes x J positions resolve the logical misses [0, count): longer ones live at the back of s_miss
      auto run_misses = [&](auto gtag, auto jtag, int count, bool back) {
        constexpr int G = decltype(gtag)::value, J = decltype(jtag)::value;
        const int grp = tid / G, gl = tid % G;
        for (int m0 = 0; m0 < count; m0 += MODEL_THREADS / G) {
          const int mi = m0 + grp;
          const bool active0 = mi < count;
          const int k = active0 ? (back ? s_miss[SPAN - 1 - mi] : s_miss[mi]) : 0;
          const int s = active0 ? s_pt[k] : 0, e = active0 ? s_pt[k + 1] : 0;
          bool active = active0;
          if (P.t.ignore_merges) {  // models/bpe/model.rs:558-567: the whole pre-token is a vocabulary entry -> one token
            int whole = 0;
            if (active0 && gl == 0 && !is_piece(s, e)) whole = vocab_whole_word(P.t, s_byte, s, e - s, s_tok) ? 1 : 0;
            whole = __shfl_sync(0xFFFFFFFFu, whole, lane & ~(G - 1));
            active = active0 && !whole;
          }
          coop_bpe<G, J>(P.t, s_byte, s_tok, s, e, active, gl);
          __syncwarp();
          // long numbers rarely repeat: publishing them only fills the table
          const bool numeric = active0 && (e - s) >= 5 && (unsigned)(s_byte[s + 1] - '0') < 10u && (unsigned)(s_byte[e - 1] - '0') < 10u;
          if (P.wcache_on && active0 && gl == 0 && e - s <= WC_MAX_BYTES && !numeric && !(P.t.ignore_merges && is_piece(s, e))) {
            WordKey key;
            wc_make_key(s_byte, s, e - s, key);
            wc_publish(P.wcache, P.wcache_mask, key, s, e, s_tok);
          }
        }
      };
      // longer pre-tokens (17..32 bytes: rare, many rounds) by lane groups
      run_misses(IntTag<8>{}, IntTag<THREAD_PATH_MAX / 8>{}, n_longer, true);
      // short ones (<= 16 bytes: nearly all misses) with fewer positions per lane.  (One THREAD per short miss, 32 words per
      // warp with the pair ranks in shared memory, needs 4-5x fewer instructions per word but was slower when tried, with the
      // cache on and off: the page waits for its longest chain of dependent probes, and a lane group's chain is the shortest.)
      run_misses(IntTag<P4_SHORT_G>{}, IntTag<(P4_SPLIT_BYTES + P4_SHORT_G - 1) / P4_SHORT_G>{}, n_short, false);
    }
    // -------------------------------------------------------------- P4b: one warp per longer pre-token (33..256 bytes)
    {
      const int nmq = s_nmq;
      for (int qi = warp; qi < nmq; qi += NWARPS) {
        const int k = s_mq[qi], s = s_pt[k], e = s_pt[k + 1];
        bool active = true;
        if (P.t.ignore_merges) {
          int whole = 0;
          if (lane == 0 && !is_piece(s, e)) whole = vocab_whole_word(P.t, s_byte, s, e - s, s_tok) ? 1 : 0;
          whole = __shfl_sync(0xFFFFFFFFu, whole, 0);
          active = !whole;
        }
        coop_bpe<32, LONG_PRETOK_MIN / 32>(P.t, s_byte, s_tok, s, e, active, lane);
      }
    }
  } else {
    // -------------------------------------------------------------- WordPiece P3: word cache, one split per thread
    for (int k0 = 0; k0 < Pproc; k0 += MODEL_THREADS) {
      const int k = k0 + tid;
      bool miss = false;
      if (k < Pproc) {
        const int s = s_pt[k], e = s_pt[k + 1], len = e - s;
        if (added_at(s)) s_tok[s] = tok_pack(added_id(s), len);
        else if ((s_keptb[s >> 5] >> (s & 31)) & 1u) {  // not removed whitespace
          bool hit = false;
          if (P.wcache_on && len <= WC_MAX_BYTES) {
            WordKey key;
            wc_make_key(s_byte, s, len, key);
            hit = wc_lookup(P.wcache, P.wcache_mask, key, s, s_tok);
          }
          miss = !hit;
        }
      }
      const unsigned mm = __ballot_sync(0xFFFFFFFFu, miss);
      int bm = 0;
      if (lane == 0 && mm) bm = atomicAdd(&s_nmiss, __popc(mm));
      bm = __shfl_sync(0xFFFFFFFFu, bm, 0);
      if (miss) s_miss[bm + __popc(mm & ((1u << lane) - 1u))] = (uint16_t)k;
    }
    __syncthreads();
    // -------------------------------------------------------------- WordPiece P4: misses, one thread per split
    const int nmiss = s_nmiss;
    while (true) {
      const int mi = atomicAdd(&s_next, 1);
      if (mi >= nmiss) break;
      const int k = s_miss[mi];
      const int s = s_pt[k], e = s_pt[k + 1], len = e - s;
      // chars = lead bytes in [s, e)
      int chars = (int)s_lpref[(e - 1) >> 5] + __popc(s_leadb[(e - 1) >> 5] & mask_le((e - 1) & 31)) -
                  ((int)s_lpref[s >> 5] + __popc(s_leadb[s >> 5] & (mask_le(s & 31) >> 1)));
      bool bad = chars > (int)P.t.max_chars;
      if (!bad) {
        int start = s;
        while (start < e) {
          uint32_t node = (start == s) ? 0u : 1u, best_id = 0;
          int best_end = -1;
          for (int p = start; p < e; ++p) {
            const uint32_t key = (node << 8) | s_byte[p];
            uint32_t slot = edge_hash(node, s_byte[p]) & P.t.edge_mask;
            uint4 en;
            while (true) {
              en = __ldg(P.t.edge_tbl + slot);
              if (en.x == key || en.x == EMPTY_KEY) break;
              slot = (slot + 1) & P.t.edge_mask;
            }
            if (en.x == EMPTY_KEY) break;
            node = en.y;
            if (en.z != EMPTY_KEY) { best_id = en.z; best_end = p + 1; }
          }
          if (best_end < 0) { bad = true; break; }
          s_tok[start] = tok_pack(best_id, best_end - start);
          start = best_end;
        }
      }
      if (bad) {
        for (int p = s; p < e; ++p) s_tok[p] = 0u;
        s_tok[s] = tok_pack(P.t.unk_id, len);
      }
      if (P.wcache_on && len <= WC_MAX_BYTES) {
        WordKey key;
        wc_make_key(s_byte, s, len, key);
        wc_publish(P.wcache, P.wcache_mask, key, s, e, s_tok);
      }
    }
    // a LONG split (> 416 bytes) has more than max_input_chars_per_word (<= 100 * 4 bytes) characters: it is [UNK];
    // count its characters for the end offset
    if (is_long) {
      const int64_t ls = base + s_pt[Pn - 1], le = s_long_end;
      int cnt = 0;
      for (int64_t p = ls + tid; p < le; p += MODEL_THREADS) cnt += ((__ldg(P.bytes + p) & 0xC0u) != 0x80u);
#pragma unroll
      for (int sft = 16; sft >= 1; sft >>= 1) cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, sft);
      if (lane == 0) atomicAdd(&s_long_chars, cnt);
    }
  }
  __syncthreads();

  // ---------------------------------------------------------------- P5: token bitmap and count
  for (int row = warp; row < NW; row += NWARPS) {
    int pos = row * 32 + lane;
    bool tok = pos >= first && pos < Eproc && tok_len(s_tok[pos]) != 0;
    uint32_t tb = __ballot_sync(0xFFFFFFFFu, tok);
    if (lane == 0) s_tokb[row] = tb;
  }
  __syncthreads();
  const bool long_kept = MODEL == MODEL_WORDPIECE && is_long && ((s_keptb[s_pt[Pn - 1] >> 5] >> (s_pt[Pn - 1] & 31)) & 1u);
  if (warp == 0) {
    int tot = warp_prefix_words(s_tokb, s_tpref, NW, lane);
    if (lane == 0) s_ntok = tot;
  }
  __syncthreads();
  {
    // compact list of token positions
    for (int row = warp; row < NW; row += NWARPS) {
      const uint32_t tb = s_tokb[row];
      if ((tb >> lane) & 1u) s_tokpos[s_tpref[row] + __popc(tb & ((1u << lane) - 1u))] = (uint16_t)(row * 32 + lane);
    }
    // ---------------------------------------------------------------- P6: page token count (no ordering between pages:
    // an in-order look-back chain stalls every page behind the slowest of the pages in flight)
    if (tid == 0) {
      const int A = s_ntok + ((MODEL == MODEL_WORDPIECE && long_kept) ? 1 : 0) + (MODEL == MODEL_BPE ? s_lcum[n_longs] : 0);
      s_ntot = A;
      s_excl = (unsigned long long)(base + first);  // provisional slot of the page's first token
      P.tile_count[t] = (uint32_t)A;
      P.tile_first[t] = (uint32_t)(base + first);
    }
  }
  __syncthreads();
  const unsigned long long excl = s_excl;
  // chars / kept splits of the document that spans into this page, counted from its start (pretok_kernels.cuh K1b)
  const uint64_t carry = __ldg(P.page_carry + t);
  int carry_chars = (int)((uint32_t)carry & 0x7FFFFFFFu), carry_starts = (int)(uint32_t)(carry >> 32);
  if (!((carry >> 31) & 1ull)) {  // no document start earlier in this scan block: add the block's carry
    const uint64_t bc = __ldg(P.block_carry + (t >> 10));
    carry_chars += (int)(uint32_t)bc; carry_starts += (int)(uint32_t)(bc >> 32);
  }
  const bool want_off = P.flags & F_OFFSETS, want_wid = P.flags & F_WORD_IDS, byte_off = P.flags & F_BYTE_OFFSETS;

  // ---------------------------------------------------------------- P7: emit tokens in order
  auto lc_incl = [&](int x) -> int { return (int)s_lpref[x >> 5] + __popc(s_leadb[x >> 5] & mask_le(x & 31)); };
  auto kept_incl = [&](int x) -> int { return (int)s_spref[x >> 5] + __popc(s_keptb[x >> 5] & mask_le(x & 31)); };
  auto doc_base = [&](int x) -> int {  // last doc start at or before x inside the page, or -1
    int xx = x < TILE ? x : TILE - 1;
    uint32_t m = s_dsb[xx >> 5] & mask_le(xx & 31);
    return m ? (xx & ~31) + 31 - __clz((int)m) : (int)s_dlast[xx >> 5];
  };
  auto emit = [&](unsigned long long out, uint32_t id, int ts, int64_t tend_abs, int end_chars_in_page, bool end_known) {
    // ts: token start (page-relative); tend_abs: absolute end byte; end_chars_in_page: lc_incl(e-1) if end_known
    P.ids[out] = (P.flag_added && ts < TILE && added_at(ts)) ? (id | 0x80000000u) : id;
    const int D = doc_base(ts);
    if (want_off) {
      uint32_t o0, o1;
      if (!byte_off) {
        const int cb = D >= 0 ? lc_incl(D) - 1 : -carry_chars;  // chars before the doc start, page-relative
        o0 = (uint32_t)(lc_incl(ts) - 1 - cb);
        o1 = (uint32_t)(end_chars_in_page - cb);
      } else {
        int64_t ds = D >= 0 ? base + D : s_span_doc_start;
        int64_t gs = base + ts, ge = tend_abs;
        while (gs > 0 && (__ldg(P.bytes + gs) & 0xC0u) == 0x80u) --gs;
        while (ge < n && (__ldg(P.bytes + ge) & 0xC0u) == 0x80u) ++ge;
        o0 = (uint32_t)(gs - ds); o1 = (uint32_t)(ge - ds);
      }
      (void)end_known;
      if (P.prefix_bits) {  // offsets were computed on the document WITH its inserted space: map back (normalizer.rs:503-514)
        const int64_t dsa = D >= 0 ? base + D : s_span_doc_start;
        if ((__ldg(P.prefix_bits + (dsa >> 5)) >> (dsa & 31)) & 1u) {
          if (o1 == 1u && byte_off) {  // the token is the inserted space alone: it is aligned to the whole first character
            int64_t ge2 = dsa + 2;
            while (ge2 < n && (__ldg(P.bytes + ge2) & 0xC0u) == 0x80u) ++ge2;
            o1 = (uint32_t)(ge2 - dsa);
          }
          o0 = o0 ? o0 - 1u : 0u;
          o1 = o1 > 2u ? o1 - 1u : 1u;
          if (byte_off && o1 < 1u) o1 = 1u;
        }
      }
      reinterpret_cast<uint2*>(P.offsets)[out] = make_uint2(o0, o1);
    }
    if (want_wid) {
      // kept splits before the doc start (the split AT the doc start may itself be removed whitespace)
      const int wb = D >= 0 ? kept_incl(D) - (int)((s_keptb[D >> 5] >> (D & 31)) & 1u) : -carry_starts;
      P.word_ids[out] = (uint32_t)(kept_incl(ts) - 1 - wb);
    }
  };
  const int n_normal = s_ntok;
  for (int j = tid; j < n_normal; j += MODEL_THREADS) {
    const int pos = s_tokpos[j];
    const unsigned long long out = excl + (unsigned long long)(j + long_tokens_before(pos));
    const uint32_t tk = s_tok[pos];
    const int e = pos + tok_len(tk);
    emit(out, tok_id(tk), pos, base + e, lc_incl(e - 1), true);
  }
  if (MODEL == MODEL_BPE) {
    // tokens of the long pre-tokens, produced by the pre-pass (relative to the pre-token start)
    for (int a = 0; a < n_longs; ++a) {
      const int ls = s_pt[s_lk[a]];
      const int ntl = s_lcum[a + 1] - s_lcum[a];
      if (ntl == 0) continue;
      const uint4* __restrict__ lo = P.long_out + s_loff[a];
      const int nb = ls == 0 ? 0 : (int)s_tpref[(ls - 1) >> 5] + __popc(s_tokb[(ls - 1) >> 5] & mask_le((ls - 1) & 31));
      const unsigned long long obase = excl + (unsigned long long)(nb + s_lcum[a]);
      const int D = doc_base(ls);
      const int cb = D >= 0 ? lc_incl(D) - 1 : -carry_chars;
      const int X = lc_incl(ls) - 1 - cb;  // char index of the pre-token's first char inside its document
      const int wb = D >= 0 ? kept_incl(D) - (int)((s_keptb[D >> 5] >> (D & 31)) & 1u) : -carry_starts;
      const uint32_t wid = (uint32_t)(kept_incl(ls) - 1 - wb);
      const int64_t ds = D >= 0 ? base + D : s_span_doc_start;
      for (int k = tid; k < ntl; k += MODEL_THREADS) {
        const uint4 r = lo[k];
        P.ids[obase + k] = r.x;
        if (want_off) {
          uint32_t o0, o1;
          if (!byte_off) { o0 = (uint32_t)X + r.z; o1 = (uint32_t)X + r.w; }
          else {
            int64_t gs = base + ls + (k ? (int64_t)lo[k - 1].y : 0), ge = base + ls + (int64_t)r.y;
            while (gs > 0 && (__ldg(P.bytes + gs) & 0xC0u) == 0x80u) --gs;
            while (ge < n && (__ldg(P.bytes + ge) & 0xC0u) == 0x80u) ++ge;
            o0 = (uint32_t)(gs - ds); o1 = (uint32_t)(ge - ds);
          }
          if (P.prefix_bits && ((__ldg(P.prefix_bits + (ds >> 5)) >> (ds & 31)) & 1u)) {
            if (o1 == 1u && byte_off) {
              int64_t ge2 = ds + 2;
              while (ge2 < n && (__ldg(P.bytes + ge2) & 0xC0u) == 0x80u) ++ge2;
              o1 = (uint32_t)(ge2 - ds);
            }
            o0 = o0 ? o0 - 1u : 0u;
            o1 = o1 > 2u ? o1 - 1u : 1u;
          }
          reinterpret_cast<uint2*>(P.offsets)[obase + k] = make_uint2(o0, o1);
        }
        if (want_wid) P.word_ids[obase + k] = wid;
      }
    }
  }
  if (MODEL == MODEL_WORDPIECE && long_kept && tid == 0) {
    const int ls = s_pt[Pn - 1];
    const unsigned long long out = excl + (unsigned long long)(s_ntot - 1);
    // chars up to the end of the long split = chars before it in the page + its own
    const int end_chars = lc_incl(ls) - 1 + s_long_chars;
    emit(out, P.t.unk_id, ls, s_long_end, end_chars, true);
  }

  // ---------------------------------------------------------------- P8: row_ptr of the documents starting in this page
  {
    const uint32_t fd = __ldg(P.page_first_doc + t);
    for (uint64_t d = (uint64_t)fd + tid; d <= P.n_docs; d += MODEL_THREADS) {
      const int64_t pos = (int64_t)__ldg(P.doc_off + d) - base;
      if (pos >= TILE) break;
      // tokens that start before `pos` (a doc start is a pre-token start, so no token straddles it)
      const int before = pos == 0 ? 0 : (int)s_tpref[(pos - 1) >> 5] + __popc(s_tokb[(pos - 1) >> 5] & mask_le((int)((pos - 1) & 31)));
      P.row_ptr[d] = (unsigned long long)(before + long_tokens_before((int)pos));  // page-local; row_ptr_fix_kernel adds the page's base
    }
  }
}


// ------------------------------------------------------------------------------------------------ pass 2
// Exclusive scan of the page token counts (two levels of 1024), then compaction of the provisional slots.
constexpr int TSCAN = 1024;

__global__ void __launch_bounds__(TSCAN) tile_scan_block_kernel(const uint32_t* __restrict__ cnt, unsigned long long* __restrict__ local_excl,
                                                                unsigned long long* __restrict__ block_sum, int64_t n_tiles) {
  __shared__ unsigned long long s_w[32];
  const int64_t i = (int64_t)blockIdx.x * TSCAN + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned long long v = i < n_tiles ? (unsigned long long)cnt[i] : 0ull;
  unsigned long long inc = v;
#pragma unroll
  for (int s = 1; s < 32; s <<= 1) { unsigned long long o = __shfl_up_sync(0xFFFFFFFFu, inc, s); if (lane >= s) inc += o; }
  if (lane == 31) s_w[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    unsigned long long w = s_w[lane], wi = w;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) { unsigned long long o = __shfl_up_sync(0xFFFFFFFFu, wi, s); if (lane >= s) wi += o; }
    s_w[lane] = wi - w;
    if (lane == 31) block_sum[blockIdx.x] = wi;
  }
  __syncthreads();
  if (i < n_tiles) local_excl[i] = s_w[warp] + inc - v;
}

__global__ void __launch_bounds__(TSCAN) tile_scan_top_kernel(unsigned long long* __restrict__ block_sum, int64_t n_blocks, unsigned long long* __restrict__ total) {
  __shared__ unsigned long long s_w[32];
  __shared__ unsigned long long s_run;
  if (threadIdx.x == 0) s_run = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t b0 = 0; b0 < n_blocks; b0 += TSCAN) {
    const int64_t i = b0 + threadIdx.x;
    const unsigned long long v = i < n_blocks ? block_sum[i] : 0ull;
    unsigned long long inc = v;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) { unsigned long long o = __shfl_up_sync(0xFFFFFFFFu, inc, s); if (lane >= s) inc += o; }
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      unsigned long long w = s_w[lane], wi = w;
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) { unsigned long long o = __shfl_up_sync(0xFFFFFFFFu, wi, s); if (lane >= s) wi += o; }
      s_w[lane] = wi - w;
    }
    __syncthreads();
    const unsigned long long run = s_run;
    if (i < n_blocks) block_sum[i] = run + s_w[warp] + inc - v;  // exclusive, in place
    __syncthreads();
    if (threadIdx.x == TSCAN - 1) s_run = run + s_w[warp] + inc;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = s_run;
}

// one warp per page: provisional slots -> final CSR positions
__global__ void compact_kernel(const uint32_t* __restrict__ tile_count, const uint32_t* __restrict__ tile_first,
                               const unsigned long long* __restrict__ local_excl, const unsigned long long* __restrict__ block_excl, int64_t n_tiles,
                               const uint32_t* __restrict__ t_ids, const uint2* __restrict__ t_off, const uint32_t* __restrict__ t_wid,
                               uint32_t* __restrict__ ids, uint2* __restrict__ off, uint32_t* __restrict__ wid) {
  const int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= n_tiles) return;
  const uint32_t cnt = tile_count[t];
  if (!cnt) return;
  const unsigned long long src = tile_first[t], dst = local_excl[t] + block_excl[t / TSCAN];
  for (uint32_t j = lane; j < cnt; j += 32) {
    ids[dst + j] = t_ids[src + j];
    if (off) off[dst + j] = t_off[src + j];
    if (wid) wid[dst + j] = t_wid[src + j];
  }
}

__global__ void row_ptr_fix_kernel(const uint64_t* __restrict__ doc_off, uint32_t n_docs, const unsigned long long* __restrict__ local_excl,
                                   const unsigned long long* __restrict__ block_excl, const uint64_t* __restrict__ row_ptr_local,
                                   uint64_t* __restrict__ row_ptr_out, unsigned long long token_base) {
  const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d > n_docs) return;
  const int64_t t = (int64_t)(doc_off[d] / TILE);
  row_ptr_out[d] = row_ptr_local[d] + local_excl[t] + block_excl[t / TSCAN] + token_base;
}

}  // namespace b2t
