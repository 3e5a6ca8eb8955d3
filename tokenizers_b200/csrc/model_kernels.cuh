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
#include <type_traits>
#include <utility>
#include "b2t_tables.h"
#include "added_kernels.cuh"
#include "long_kernels.cuh"
#include "pretok_logic.cuh"

namespace b2t {

constexpr int TILE = PAGE;
constexpr int MODEL_THREADS = 256;
constexpr int THREAD_PATH_MAX = 32;  // pre-tokens up to this many bytes are merged by an 8-lane group, longer ones by a warp
enum { MODEL_BPE = 0, MODEL_WORDPIECE = 1 };
constexpr int MAX_LONG_PER_PAGE = TILE / (LONG_PRETOK_MIN + 1) + 1;  // 8

// What a call writes per token, a template parameter of the page kernel: offsets (char offsets unless L_BYTE_OFFSETS),
// word ids, the mapping of offsets back across an inserted prefix space (L_PREFIX), bit 31 on the ids of added tokens
// (L_ADDED_IDS).  Each layout is an instance of its own, so code for outputs a call does not want takes no registers
// (one instance with runtime flags ran at 32 registers with spills).  MODEL_LAYOUTS lists every mask a call can form:
// byte offsets and the prefix mapping only come with offsets.
enum : unsigned { L_OFFSETS = 1u, L_WORD_IDS = 2u, L_BYTE_OFFSETS = 4u, L_PREFIX = 8u, L_ADDED_IDS = 16u };
constexpr unsigned MODEL_LAYOUTS[] = {0u, 1u, 5u, 9u, 13u, 2u, 3u, 7u, 11u, 15u, 16u, 17u, 21u, 25u, 29u, 18u, 19u, 23u, 27u, 31u};
constexpr int N_MODEL_LAYOUTS = (int)(sizeof(MODEL_LAYOUTS) / sizeof(MODEL_LAYOUTS[0]));
constexpr int model_layout_index(unsigned lay) {
  for (int i = 0; i < N_MODEL_LAYOUTS; ++i)
    if (MODEL_LAYOUTS[i] == lay) return i;
  return -1;
}

struct ModelParams {
  const uint8_t* bytes; int64_t n;
  const uint32_t* start_bits; const uint32_t* drop_bits; const uint32_t* doc_bits;
  // BPE: exact cuts inside long pre-tokens (long_kernels.cuh soft_cut) and the pages that hold any; the page kernel merges
  // the pieces like pre-tokens of their own, word ids and offsets keep following start_bits
  const uint32_t* soft_bits; const uint8_t* page_soft;
  const uint64_t* page_carry; const uint64_t* block_carry; const uint32_t* page_first_doc;
  const uint64_t* doc_off; uint32_t n_docs;
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
  // the page; NULL when the batch did not go through the extraction.  (L_ADDED_IDS: mark those tokens with bit 31 of the id.)
  const uint32_t* added_bits; const uint32_t* added_head; const uint2* added_pool;
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

// exclusive prefix of popcounts over nw (<= 96) words, by one full warp (lane writes pref[3 lane .. 3 lane + 2]); returns
// the total
template <class T>
__device__ __forceinline__ int warp_prefix_words(const uint32_t* bits, T* pref, int nw, int lane) {
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
  if (i < nw) pref[i] = (T)ex;
  if (i + 1 < nw) pref[i + 1] = (T)(ex + c0);
  if (i + 2 < nw) pref[i + 2] = (T)(ex + c0 + c1);
  return __shfl_sync(0xFFFFFFFFu, inc, 31);
}

__device__ __forceinline__ uint32_t mask_le(int b) { return b >= 31 ? 0xFFFFFFFFu : ((2u << b) - 1u); }
__device__ __forceinline__ uint32_t mask_lt(int b) { return (1u << b) - 1u; }   // b in [0, 32)

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
#ifdef B2T_WC_TEST_FP_MASK   // the host build in tests/native only: fingerprints that collide on purpose, so a hit rests on the key compare
  key.fp = (key.fp & B2T_WC_TEST_FP_MASK) ? (key.fp & B2T_WC_TEST_FP_MASK) : 1ull;
#endif
}

// Memory-model note.  A slot is written once per batch (the table is zeroed, stream-ordered, before the kernel) and never
// changes after that, readers take no lock and no fence -- an acquire load costs an L1 invalidation (CCTL.IVALL) per
// probe on this architecture, and the merge-table probes live in L1.  Instead every 32-bit word of a written slot is
// NON-ZERO by construction (key words and ids are stored complemented: a key word of 0xFFFFFFFF cannot occur in UTF-8,
// ids are < 2^20; the two length words carry a marker bit), all accesses are strong (.relaxed.gpu, single-copy atomic
// per 32-bit word), and a reader accepts a slot only if the words it uses are non-zero and the whole key matches.  A word
// that is not yet visible reads as zero, which is a miss: the pre-token is merged, the result is the same.
// (The host branches serve the host build of the kernels in tests/native: the PTX memory model treats a vector access as
// one access per element, so per-word relaxed atomics are the same thing.)
__device__ __forceinline__ uint4 ld_relaxed_v4(const uint4* p) {
  uint4 v;
#ifdef __CUDA_ARCH__
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
#else
  v.x = __atomic_load_n(&p->x, __ATOMIC_RELAXED); v.y = __atomic_load_n(&p->y, __ATOMIC_RELAXED);
  v.z = __atomic_load_n(&p->z, __ATOMIC_RELAXED); v.w = __atomic_load_n(&p->w, __ATOMIC_RELAXED);
#endif
  return v;
}
__device__ __forceinline__ void st_relaxed_v4(uint4* p, uint4 v) {
#ifdef __CUDA_ARCH__
  asm volatile("st.relaxed.gpu.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
#else
  __atomic_store_n(&p->x, v.x, __ATOMIC_RELAXED); __atomic_store_n(&p->y, v.y, __ATOMIC_RELAXED);
  __atomic_store_n(&p->z, v.z, __ATOMIC_RELAXED); __atomic_store_n(&p->w, v.w, __ATOMIC_RELAXED);
#endif
}
constexpr uint32_t WC_LEN_MARK = 0x80000000u;   // bit 31 of the second length word: always set in a written slot

// Looks up the pre-token [s, s + len) unless the cache is off, it is too long or the caller has a reason to `skip` it.
// Returns true on a hit (tokens written to s_tok).
__device__ __forceinline__ bool wc_lookup(const ModelParams& P, const uint8_t* s_byte, uint32_t* s_tok, int s, int len, bool skip) {
  if (!P.wcache_on || len > WC_MAX_BYTES || skip) return false;
  WordKey key;
  wc_make_key(s_byte, s, len, key);
  const uint4* cache = P.wcache;
  const uint32_t mask = P.wcache_mask;
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
    const uint4 q2 = ld_relaxed_v4(q + 2);
    const int ntok = (int)(q2.x & 0xFFu);
    // ids 2..5 only for words that have them (most have one or two tokens): the look-ups pay per L2 request, not per
    // byte -- on an H100 at 700 W, one more load per look-up (the key together with the tag, same sector) cost bpe_tile 10 %
    const uint4 q3 = ntok > 2 ? ld_relaxed_v4(q + 3) : make_uint4(0u, 0u, 0u, 0u);
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

// Publish the merged pre-token [s, e) (symbols chained by their lengths) into the first free slot of its probe sequence,
// under the same conditions as wc_lookup.
__device__ __forceinline__ void wc_publish(const ModelParams& P, const uint8_t* s_byte, const uint32_t* s_tok, int s, int e, bool skip) {
  if (!P.wcache_on || e - s > WC_MAX_BYTES || skip) return;
  WordKey key;
  wc_make_key(s_byte, s, e - s, key);
  uint4* const cache = P.wcache;
  const uint32_t mask = P.wcache_mask;
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
#ifdef __CUDA_ARCH__
      asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1, %2};" ::"l"(kw + 2), "r"(~key.k[0]), "r"(~key.k[1]) : "memory");
#else
      __atomic_store_n(kw + 2, ~key.k[0], __ATOMIC_RELAXED); __atomic_store_n(kw + 3, ~key.k[1], __ATOMIC_RELAXED);
#endif
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


// ------------------------------------------------------------------------------------------------ page state
// Set bits of `bits` at positions <= x; pref[w] = set bits in the words before w.
__device__ __forceinline__ int bit_rank_incl(const uint16_t* pref, const uint32_t* bits, int x) {
  return (int)pref[x >> 5] + __popc(bits[x >> 5] & mask_le(x & 31));
}
__device__ __forceinline__ bool bit_at(const uint32_t* bits, int x) { return (bits[x >> 5] >> (x & 31)) & 1u; }

// Shared memory of one page, laid out without padding.  byte / tok: the page + halo and the token starting at each
// position (tok_pack).  Bitmaps, one bit per position: startb = units of merging (splits of the pre-tokenizer + exact
// cuts of long ones), keptb = splits the reference keeps (word ids), leadb = first bytes of characters, tokb = token
// starts, dsb = document starts, addedb = added-token spans; apref / spref / lpref = exclusive prefix of the popcounts of
// startb / keptb / leadb per word; tpref = the page's tokens before each word, the long pre-tokens' included (a long
// pre-token covers the rest of its word, so its tokens come after every token of that word and before the next word's).
// Per word of the page, the document in force at its first position: dlast = its start, or -1 when it began in an
// earlier page; dcb / dwb = chars / kept splits of the page before that start (negative: the carry of the earlier
// pages, carry_c / carry_w).  pt: the page's pre-token starts, then the end of the last one.  list: pre-tokens the word
// cache did not resolve.  BPE: mq = pre-tokens of 33..256 bytes; lk / lcum / loff = the long pre-tokens starting in the
// page (indices in position order, exclusive prefix of their token counts, place in long_out).
template <int HALO_>
struct PageCommon {
  static constexpr int HALO = HALO_, SPAN = TILE + HALO, NW = SPAN / 32, TW = TILE / 32;
  static_assert(NW <= 96 && SPAN % 16 == 0, "warp_prefix_words handles <= 96 words; tok is 16-byte aligned");
  static_assert(2 * TW <= MODEL_THREADS, "stage_page: one thread per word of the page for pt, one for dcb / dwb");
  uint8_t byte[SPAN];
  uint32_t tok[SPAN];
  long long span_doc_start;  // first byte of the document that spans into this page
  uint32_t startb[NW + 1], keptb[NW + 1], leadb[NW + 1], tokb[NW + 1], dsb[TW + 1], addedb[TW + 1];
  int tpref[NW + 1], dcb[TW], dwb[TW];
  uint16_t apref[NW + 1], spref[NW + 1], lpref[NW + 1];
  int16_t dlast[TW + 1];
  uint16_t pt[TILE + 2], list[SPAN];
  int tile, npt, elast, is_long, ntok, nmiss, carry_c, carry_w;
};
struct BpePage : PageCommon<256> {
  uint16_t mq[TILE / THREAD_PATH_MAX + 2], lk[MAX_LONG_PER_PAGE + 1];
  int nmiss_hi, nmq, anysoft, nl, lcum[MAX_LONG_PER_PAGE + 2];  // nmiss_hi: misses queued from the back of list
  unsigned long long loff[MAX_LONG_PER_PAGE + 1];
};
struct WpPage : PageCommon<416> {
  long long long_end;  // end of a split that runs past the halo
  int next, long_chars;
};
template <int MODEL> using PageState = std::conditional_t<MODEL == MODEL_BPE, BpePage, WpPage>;

// [s, e) is a piece of a cut pre-token (not a whole split of the pre-tokenizer): with ignore_merges the whole-word rule
// and the word cache (whose entries follow that rule) do not apply to it
__device__ __forceinline__ bool is_piece(const BpePage& sh, int64_t base, int64_t n, int s, int e) {
  if (!sh.anysoft) return false;
  const bool real_e = base + e >= n || (e < BpePage::SPAN && bit_at(sh.keptb, e));
  return !(bit_at(sh.keptb, s) && real_e);
}

// the pre-token that starts at s (inside the page) is an added token's span: its id comes from the page's list
template <class S>
__device__ __forceinline__ bool added_at(const ModelParams& P, const S& sh, int s) { return P.added_bits != nullptr && bit_at(sh.addedb, s); }
__device__ __forceinline__ uint32_t added_id(const ModelParams& P, int64_t t, int s) {
  for (uint32_t i = __ldg(P.added_head + t); i != ADDED_NIL;) {
    const uint2 v = __ldg(P.added_pool + i);
    if ((int)(v.x & (uint32_t)(PAGE - 1)) == s) return v.x >> 11;
    i = v.y;
  }
  atomicOr(P.err_flag, ERR_INTERNAL);
  return 0u;
}

// Warp-aggregated append of k, for the lanes with `take`, to the queue q of length *len: one shared atomic per warp.
// back: the queue grows downwards from q.
__device__ __forceinline__ void warp_enqueue(uint16_t* q, int* len, bool take, int k, bool back) {
  const int lane = threadIdx.x & 31;
  const unsigned m = __ballot_sync(0xFFFFFFFFu, take);
  int b = 0;
  if (lane == 0 && m) b = atomicAdd(len, __popc(m));
  b = __shfl_sync(0xFFFFFFFFu, b, 0) + __popc(m & ((1u << lane) - 1u));
  if (take) q[back ? -b : b] = (uint16_t)k;
}

// models/bpe/model.rs:558-567 (ignore_merges): a vocabulary entry is one token.  Called by all 32 lanes (a shuffle):
// the lane with `ask` looks the pre-token up, every lane learns from lane `leader` whether its group skips the merge.
__device__ __forceinline__ bool whole_word_gate(const ModelParams& P, const uint8_t* s_byte, uint32_t* s_tok, int s, int e, bool ask, int leader) {
  if (!P.t.ignore_merges) return false;
  const int whole = ask && vocab_whole_word(P.t, s_byte, s, e - s, s_tok) ? 1 : 0;
  return __shfl_sync(0xFFFFFFFFu, whole, leader) != 0;
}

// g moved by `step` (-1 / +1) to the nearest character boundary of the batch
__device__ __forceinline__ int64_t char_boundary(const ModelParams& P, int64_t g, int step) {
  while ((step < 0 ? g > 0 : g < P.n) && (__ldg(P.bytes + g) & 0xC0u) == 0x80u) g += step;
  return g;
}

// Where a token's document starts, seen from the page position x where the token's pre-token starts: ds = its first
// byte, cb = chars of the page before it (negative: it started in an earlier page), wid = the pre-token's word id.
// Shared-memory reads of the facts stage_page keeps per word; only a doc start in x's own word is ranked here.
struct DocOrigin { int64_t ds; int cb; uint32_t wid; };
template <unsigned LAY, class S>
__device__ __forceinline__ DocOrigin doc_origin(const S& sh, int64_t base, int x) {
  const int xx = x < TILE ? x : TILE - 1, w = xx >> 5;
  const uint32_t m = sh.dsb[w] & mask_le(xx & 31);
  DocOrigin o;
  int wb;  // kept splits before the doc start (the split AT the doc start may itself be removed whitespace)
  if (m) {  // the last doc start at or before x is in x's word
    const int D = (xx & ~31) + 31 - __clz((int)m);
    o.ds = base + D;
    o.cb = bit_rank_incl(sh.lpref, sh.leadb, D) - 1;
    wb = bit_rank_incl(sh.spref, sh.keptb, D) - (int)bit_at(sh.keptb, D);
  } else {
    const int D = sh.dlast[w];
    o.ds = D >= 0 ? base + D : sh.span_doc_start;
    o.cb = sh.dcb[w];
    wb = sh.dwb[w];
  }
  o.wid = (LAY & L_WORD_IDS) ? (uint32_t)(bit_rank_incl(sh.spref, sh.keptb, x) - 1 - wb) : 0u;
  return o;
}

// Offsets and word id of the token in slot `out`: c0 / c1 = chars of the page before its first char / up to its end
// (for char offsets); g0 / g1 = its bytes in the batch (for byte offsets, widened to whole characters).
template <unsigned LAY>
__device__ __forceinline__ void place_token(const ModelParams& P, const DocOrigin& o, unsigned long long out,
                                            int c0, int c1, int64_t g0, int64_t g1) {
  if constexpr ((LAY & L_OFFSETS) != 0) {
    constexpr bool byte_off = (LAY & L_BYTE_OFFSETS) != 0;
    uint32_t o0, o1;
    if constexpr (!byte_off) {
      o0 = (uint32_t)(c0 - o.cb); o1 = (uint32_t)(c1 - o.cb);
    } else {
      o0 = (uint32_t)(char_boundary(P, g0, -1) - o.ds); o1 = (uint32_t)(char_boundary(P, g1, 1) - o.ds);
    }
    if constexpr ((LAY & L_PREFIX) != 0) {
      if ((__ldg(P.prefix_bits + (o.ds >> 5)) >> (o.ds & 31)) & 1u) {
        // offsets were computed on the document WITH its inserted space: map back (normalizer.rs:503-514)
        if (o1 == 1u && byte_off) o1 = (uint32_t)(char_boundary(P, o.ds + 2, 1) - o.ds);  // the space alone: its whole first character
        o0 = o0 ? o0 - 1u : 0u;
        o1 = o1 > 2u ? o1 - 1u : 1u;
      }
    }
    reinterpret_cast<uint2*>(P.offsets)[out] = make_uint2(o0, o1);
  }
  if constexpr ((LAY & L_WORD_IDS) != 0) P.word_ids[out] = o.wid;
}

// A token of the page logic (and a long WordPiece split's [UNK]) that starts at page position ts: c1 / g1 as above.
template <unsigned LAY, class S>
__device__ __forceinline__ void emit_token(const ModelParams& P, const S& sh, int64_t base, unsigned long long out,
                                           uint32_t id, int ts, int c1, int64_t g1) {
  P.ids[out] = ((LAY & L_ADDED_IDS) && ts < TILE && bit_at(sh.addedb, ts)) ? (id | 0x80000000u) : id;
  place_token<LAY>(P, doc_origin<LAY>(sh, base, ts), out, bit_rank_incl(sh.lpref, sh.leadb, ts) - 1, c1, base + ts, g1);
}

// ------------------------------------------------------------------------------------------------ page phases
// The pre-tokens the page logic resolves: pt[0, pproc), whose bytes are [first, eproc).  is_long: the page's last
// pre-token runs past the halo.  WordPiece: that split is [UNK], emitted on its own.  BPE: long pre-tokens (collected
// by collect_long_pretokens) are skipped.  Each phase reads it again: with 32 registers, a value live across phases spills.
struct PageSpan { int first, eproc, pproc; bool is_long, long_kept; };
template <int MODEL, class S>
__device__ __forceinline__ PageSpan page_span(const S& sh) {
  const int Pn = sh.npt;
  PageSpan r;
  r.is_long = sh.is_long && Pn > 0;  // without a start in the page the long pre-token belongs to an earlier page
  const bool wp_long = MODEL == MODEL_WORDPIECE && r.is_long;
  r.first = Pn ? (int)sh.pt[0] : sh.elast;
  r.eproc = Pn ? (wp_long ? (int)sh.pt[Pn - 1] : sh.elast) : 0;
  r.pproc = wp_long ? Pn - 1 : Pn;
  r.long_kept = wp_long && bit_at(sh.keptb, sh.pt[Pn - 1]);  // WordPiece: the long split is not removed whitespace
  return r;
}

// P0-P2: stage bytes and bitmaps, prefix sums, the pre-token starts
template <int MODEL, class S>
__device__ __forceinline__ void stage_page(const ModelParams& P, S& sh, int64_t t, int64_t base) {
  constexpr int SPAN = S::SPAN, NW = S::NW, TW = S::TW;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t n = P.n, n_chunks = n / CHUNK + 1;
  for (int i = tid; i < SPAN / 16; i += MODEL_THREADS) {
    int64_t g = base + (int64_t)i * 16;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (g + 16 <= n) v = __ldg(reinterpret_cast<const uint4*>(P.bytes + g));
    else if (g < n) {
      uint32_t w[4] = {0, 0, 0, 0};
      for (int k = 0; k < 16 && g + k < n; ++k) w[k >> 2] |= (uint32_t)__ldg(P.bytes + g + k) << (8 * (k & 3));
      v = make_uint4(w[0], w[1], w[2], w[3]);
    }
    reinterpret_cast<uint4*>(sh.byte)[i] = v;
  }
  for (int w = tid; w <= NW; w += MODEL_THREADS) {
    int64_t gw = base / 32 + w;
    uint32_t sb = (w < NW && gw < n_chunks) ? __ldg(P.start_bits + gw) : 0u;
    uint32_t db = (MODEL == MODEL_WORDPIECE && w < NW && gw < n_chunks) ? __ldg(P.drop_bits + gw) : 0u;
    uint32_t sf = 0u;
    if constexpr (MODEL == MODEL_BPE)
      if (w < NW && gw < n_chunks && __ldg(P.page_soft + (gw >> 6))) { sf = __ldg(P.soft_bits + gw); if (sf) sh.anysoft = 1; }
    sh.startb[w] = sb | sf;
    sh.keptb[w] = sb & ~db;
    if (w <= TW) sh.dsb[w] = (w < TW && gw < n_chunks) ? __ldg(P.doc_bits + gw) : 0u;
    if (w <= TW) sh.addedb[w] = (P.added_bits && w < TW && gw < n_chunks) ? __ldg(P.added_bits + gw) : 0u;
  }
  __syncthreads();
  // lead bits (16 bytes per thread: continuation-byte flags by SWAR, two threads make one bitmap word) + symbol init
  static_assert(SPAN / 16 <= MODEL_THREADS && (SPAN / 16) % 2 == 0, "one pass, thread pairs inside a warp");
  const int i = tid;
  const bool act = i < SPAN / 16;
  const uint4 v = act ? reinterpret_cast<const uint4*>(sh.byte)[i] : make_uint4(0u, 0u, 0u, 0u);
  const uint32_t c0 = v.x & ~(v.x << 1) & 0x80808080u, c1 = v.y & ~(v.y << 1) & 0x80808080u,
                 c2 = v.z & ~(v.z << 1) & 0x80808080u, c3 = v.w & ~(v.w << 1) & 0x80808080u;   // 10xxxxxx
  const uint32_t cont = movemask2(c0, c1) | (movemask2(c2, c3) << 8);
  const int64_t lim = n - base - (int64_t)i * 16;          // valid bytes from this thread's first position on
  const uint32_t valid = lim >= 16 ? 0xFFFFu : (lim <= 0 ? 0u : ((1u << (int)lim) - 1u));
  const uint32_t lead16 = ~cont & valid;
  const uint32_t other = __shfl_down_sync(0xFFFFFFFFu, lead16, 1);
  if (act && !(i & 1)) sh.leadb[i >> 1] = lead16 | (other << 16);
  if (act) {   // token starts are written by whoever resolves the pre-token
    uint4* z = reinterpret_cast<uint4*>(sh.tok) + 4 * i;
    z[0] = make_uint4(0u, 0u, 0u, 0u); z[1] = make_uint4(0u, 0u, 0u, 0u); z[2] = make_uint4(0u, 0u, 0u, 0u); z[3] = make_uint4(0u, 0u, 0u, 0u);
  }
  if (tid == 0) sh.leadb[NW] = 0u;
  __syncthreads();
  // prefixes, end of the last pre-token, last doc start before each word, the spanning document's start
  if (warp == 0) {
    int tot = warp_prefix_words(sh.startb, sh.apref, TW, lane);  // all starts inside the page
    if (lane == 0) sh.npt = tot;
  } else if (warp == 1) {
    warp_prefix_words(sh.keptb, sh.spref, NW, lane);
  } else if (warp == 2) {
    warp_prefix_words(sh.leadb, sh.lpref, NW, lane);
  } else if (warp == 3) {
    // first start bit at a position >= TILE (the end of the page's last pre-token)
    int found = SPAN;
    for (int w = TW + lane; w < NW; w += 32) {
      uint32_t b = sh.startb[w];
      if (b) { found = w * 32 + (__ffs((int)b) - 1); break; }
    }
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) found = min(found, __shfl_xor_sync(0xFFFFFFFFu, found, s));
    int64_t lim = n - base;  // bytes available from the page start
    int is_long = 0;
    if (found >= SPAN) {
      if (lim <= SPAN) found = (int)lim;
      else {
        // no start inside the halo: the last pre-token is LONG
        is_long = 1;
        found = SPAN;
        if constexpr (MODEL == MODEL_WORDPIECE) {  // find its true end in the global bitmap (BPE: the pre-pass knows it)
          int64_t gw = (base + SPAN) / 32;
          long long e = -1;
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
          if (lane == 0) sh.long_end = e < n ? e : n;
        }
      }
    } else if (found > lim) found = (int)lim;
    if (lane == 0) { sh.elast = found; sh.is_long = is_long; }
  } else if (warp == 4) {
    // last doc start strictly before each word of the page; lane handles words 2*lane, 2*lane+1
    uint32_t b0 = sh.dsb[2 * lane], b1 = sh.dsb[2 * lane + 1];
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
    sh.dlast[2 * lane] = (int16_t)before; sh.dlast[2 * lane + 1] = (int16_t)max(before, last0);
    if (lane == 31) sh.dlast[TW] = (int16_t)inc;
  } else if (warp == 5 && lane == 0) {
    uint32_t fd = __ldg(P.page_first_doc + t);
    sh.span_doc_start = fd > 0 ? (long long)__ldg(P.doc_off + fd - 1) : 0;
    // chars / kept splits of the document before this page, counted from its start (pretok_kernels.cuh K1b), + the scan
    // block's carry
    const uint64_t c = __ldg(P.page_carry + t);
    const uint64_t bc = (c >> 31) & 1ull ? 0ull : __ldg(P.block_carry + (t >> 10));
    sh.carry_c = (int)(((uint32_t)c & 0x7FFFFFFFu) + (uint32_t)bc);
    sh.carry_w = (int)((uint32_t)(c >> 32) + (uint32_t)(bc >> 32));
  }
  __syncthreads();
  if (tid < TW) {
    uint32_t bits = sh.startb[tid];
    int idx = sh.apref[tid];
    while (bits) { sh.pt[idx++] = (uint16_t)(tid * 32 + __ffs((int)bits) - 1); bits &= bits - 1u; }
  } else if (tid < 2 * TW) {  // the document in force at the first position of word w (doc_origin)
    const int w = tid - TW, D = sh.dlast[w];
    sh.dcb[w] = D >= 0 ? bit_rank_incl(sh.lpref, sh.leadb, D) - 1 : -sh.carry_c;
    sh.dwb[w] = D >= 0 ? bit_rank_incl(sh.spref, sh.keptb, D) - (int)bit_at(sh.keptb, D) : -sh.carry_w;
  }
  if (tid == 0) sh.pt[sh.npt] = (uint16_t)sh.elast;
}

// BPE: pre-tokens longer than LONG_PRETOK_MIN were resolved by the pre-pass; collect them (position order) and clear
// their symbols so that the page logic skips them
__device__ __forceinline__ void collect_long_pretokens(const ModelParams& P, BpePage& sh, int64_t t, int64_t base) {
  const int tid = threadIdx.x, Pn = sh.npt;
  int any_long = 0;
  for (int k = tid; k < Pn; k += MODEL_THREADS)
    if ((int)sh.pt[k + 1] - (int)sh.pt[k] > LONG_PRETOK_MIN) { int i = atomicAdd(&sh.nl, 1); if (i < MAX_LONG_PER_PAGE) sh.lk[i] = (uint16_t)k; any_long = 1; }
  if (!__syncthreads_or(any_long)) return;   // (almost every page: no long pre-token, one barrier instead of three)
  if (tid == 0) {
    int nl = sh.nl;
    if (nl > MAX_LONG_PER_PAGE) { nl = MAX_LONG_PER_PAGE; atomicOr(P.err_flag, ERR_INTERNAL); }
    for (int a = 1; a < nl; ++a) { uint16_t v = sh.lk[a]; int b = a - 1; while (b >= 0 && sh.lk[b] > v) { sh.lk[b + 1] = sh.lk[b]; --b; } sh.lk[b + 1] = v; }
    const int32_t slot0 = nl ? __ldg(P.page_long + t) : 0;
    if (nl && slot0 < 0) { atomicOr(P.err_flag, ERR_INTERNAL); nl = 0; }
    int cum = 0;
    for (int a = 0; a < nl; ++a) {
      const LongDesc d = P.long_desc[slot0 + a];
      if (d.start != base + sh.pt[sh.lk[a]]) atomicOr(P.err_flag, ERR_INTERNAL);
      sh.lcum[a] = cum; sh.loff[a] = d.pool_off;
      cum += (d.pool_off == ~0ull) ? 0 : (int)d.ntok;
    }
    sh.lcum[nl] = cum;
    sh.nl = nl;
  }
  __syncthreads();
  for (int a = 0; a < sh.nl; ++a) {
    const int ls = sh.pt[sh.lk[a]], le = min((int)sh.pt[sh.lk[a] + 1], BpePage::SPAN);
    for (int pos = ls + tid; pos < le; pos += MODEL_THREADS) sh.tok[pos] = 0u;
  }
  __syncthreads();
}

// G lanes x J positions merge the misses [0, count) of the queue; the queue from the back of list when `back`.  count
// is read from shared memory each round: held in a register across the merges, it spills.
template <int G, int J>
__device__ __forceinline__ void merge_misses(const ModelParams& P, BpePage& sh, int64_t base, const int& count, bool back) {
  const int tid = threadIdx.x, lane = tid & 31, grp = tid / G, gl = tid % G;
  for (int m0 = 0; m0 < count; m0 += MODEL_THREADS / G) {
    const int mi = m0 + grp;
    const bool active0 = mi < count;
    const int k = active0 ? (back ? sh.list[BpePage::SPAN - 1 - mi] : sh.list[mi]) : 0;
    const int s = active0 ? sh.pt[k] : 0, e = active0 ? sh.pt[k + 1] : 0;
    const bool whole = whole_word_gate(P, sh.byte, sh.tok, s, e, active0 && gl == 0 && !is_piece(sh, base, P.n, s, e), lane & ~(G - 1));
    const bool active = active0 && !whole;
    coop_bpe<G, J>(P.t, sh.byte, sh.tok, s, e, active, gl);
    __syncwarp();
    // long numbers rarely repeat: publishing them only fills the table
    const bool numeric = active0 && (e - s) >= 5 && (unsigned)(sh.byte[s + 1] - '0') < 10u && (unsigned)(sh.byte[e - 1] - '0') < 10u;
    if (active0 && gl == 0) wc_publish(P, sh.byte, sh.tok, s, e, numeric || (P.t.ignore_merges && is_piece(sh, base, P.n, s, e)));
  }
}

// BPE P3 (word cache, one pre-token per thread), P4a (misses of <= 32 bytes, G lanes each), P4b (33..256 bytes, a warp each)
__device__ __forceinline__ void resolve_bpe(const ModelParams& P, BpePage& sh, int64_t t, int64_t base) {
  const int Pproc = page_span<MODEL_BPE>(sh).pproc;
  constexpr int SPAN = BpePage::SPAN, NWARPS = MODEL_THREADS / 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // (static assignment: a lookup costs the same for every lane, so the warp stays converged)
  for (int k0 = 0; k0 < Pproc; k0 += MODEL_THREADS) {
    const int k = k0 + tid;
    int kind = 0;  // 0 = resolved / nothing to do, 1 = miss (<= 32 bytes), 2 = medium (33..256 bytes)
    if (k < Pproc) {
      const int s = sh.pt[k], e = sh.pt[k + 1], len = e - s;
      if (added_at(P, sh, s)) sh.tok[s] = tok_pack(added_id(P, t, s), len);   // an added token: one token, whatever the model says
      else if (len > LONG_PRETOK_MIN) kind = 0;  // resolved by the pre-pass
      else if (len > THREAD_PATH_MAX) kind = 2;
      else kind = wc_lookup(P, sh.byte, sh.tok, s, len, P.t.ignore_merges && is_piece(sh, base, P.n, s, e)) ? 0 : 1;
    }
    // the four groups of a warp step through their merges together, so pre-tokens of similar length should share a
    // warp: short misses queue from the front of list, longer ones from the back
    const bool longer = kind == 1 && (int)sh.pt[k + 1] - (int)sh.pt[k] > P4_SPLIT_BYTES;
    warp_enqueue(sh.list, &sh.nmiss, kind == 1 && !longer, k, false);
    warp_enqueue(sh.list + SPAN - 1, &sh.nmiss_hi, longer, k, true);
    warp_enqueue(sh.mq, &sh.nmq, kind == 2, k, false);
  }
  __syncthreads();
  // longer pre-tokens (17..32 bytes: rare, many rounds) by lane groups
  merge_misses<8, THREAD_PATH_MAX / 8>(P, sh, base, sh.nmiss_hi, true);
  // short ones (<= 16 bytes: nearly all misses) with fewer positions per lane.  (One THREAD per short miss, 32 words per
  // warp with the pair ranks in shared memory, needs 4-5x fewer instructions per word but was slower when tried, with the
  // cache on and off: the page waits for its longest chain of dependent probes, and a lane group's chain is the shortest.)
  merge_misses<P4_SHORT_G, (P4_SPLIT_BYTES + P4_SHORT_G - 1) / P4_SHORT_G>(P, sh, base, sh.nmiss, false);
  const int nmq = sh.nmq;
  for (int qi = warp; qi < nmq; qi += NWARPS) {
    const int k = sh.mq[qi], s = sh.pt[k], e = sh.pt[k + 1];
    const bool active = !whole_word_gate(P, sh.byte, sh.tok, s, e, lane == 0 && !is_piece(sh, base, P.n, s, e), 0);
    coop_bpe<32, LONG_PRETOK_MIN / 32>(P.t, sh.byte, sh.tok, s, e, active, lane);
  }
}

// WordPiece P3 (word cache, one split per thread), P4 (misses, one thread per split), and the characters of a split
// that runs past the halo
__device__ __forceinline__ void resolve_wordpiece(const ModelParams& P, WpPage& sh, int64_t t, int64_t base) {
  const PageSpan sp = page_span<MODEL_WORDPIECE>(sh);
  const int tid = threadIdx.x, lane = tid & 31;
  for (int k0 = 0; k0 < sp.pproc; k0 += MODEL_THREADS) {
    const int k = k0 + tid;
    bool miss = false;
    if (k < sp.pproc) {
      const int s = sh.pt[k], e = sh.pt[k + 1], len = e - s;
      if (added_at(P, sh, s)) sh.tok[s] = tok_pack(added_id(P, t, s), len);
      else if (bit_at(sh.keptb, s)) miss = !wc_lookup(P, sh.byte, sh.tok, s, len, false);  // not removed whitespace
    }
    warp_enqueue(sh.list, &sh.nmiss, miss, k, false);
  }
  __syncthreads();
  const int nmiss = sh.nmiss;
  while (true) {
    const int mi = atomicAdd(&sh.next, 1);
    if (mi >= nmiss) break;
    const int k = sh.list[mi];
    const int s = sh.pt[k], e = sh.pt[k + 1], len = e - s;
    // chars = lead bytes in [s, e)
    const int chars = bit_rank_incl(sh.lpref, sh.leadb, e - 1) - (s ? bit_rank_incl(sh.lpref, sh.leadb, s - 1) : 0);
    bool bad = chars > (int)P.t.max_chars;
    if (!bad) {
      int start = s;
      while (start < e) {
        uint32_t node = (start == s) ? 0u : 1u, best_id = 0;
        int best_end = -1;
        for (int p = start; p < e; ++p) {
          const uint32_t key = (node << 8) | sh.byte[p];
          uint32_t slot = edge_hash(node, sh.byte[p]) & P.t.edge_mask;
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
        sh.tok[start] = tok_pack(best_id, best_end - start);
        start = best_end;
      }
    }
    if (bad) {
      for (int p = s; p < e; ++p) sh.tok[p] = 0u;
      sh.tok[s] = tok_pack(P.t.unk_id, len);
    }
    wc_publish(P, sh.byte, sh.tok, s, e, false);
  }
  // a LONG split (> 416 bytes) has more than max_input_chars_per_word (<= 100 * 4 bytes) characters: it is [UNK];
  // count its characters for the end offset
  if (sp.is_long) {
    const int64_t ls = base + sh.pt[sh.npt - 1], le = sh.long_end;
    int cnt = 0;
    for (int64_t p = ls + tid; p < le; p += MODEL_THREADS) cnt += ((__ldg(P.bytes + p) & 0xC0u) != 0x80u);
#pragma unroll
    for (int sft = 16; sft >= 1; sft >>= 1) cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, sft);
    if (lane == 0) atomicAdd(&sh.long_chars, cnt);
  }
}

// P5/P6: token bitmap, its prefix (long pre-tokens included) and the page's token count (no ordering between pages: an
// in-order look-back chain stalls every page behind the slowest of the pages in flight)
template <int MODEL, class S>
__device__ __forceinline__ void count_tokens(const ModelParams& P, S& sh, int64_t t, int64_t base) {
  const int tid = threadIdx.x, lane = tid & 31;
  const PageSpan sp = page_span<MODEL>(sh);
  for (int row = tid >> 5; row < S::NW; row += MODEL_THREADS / 32) {
    const int pos = row * 32 + lane;
    const uint32_t tb = __ballot_sync(0xFFFFFFFFu, pos >= sp.first && pos < sp.eproc && tok_len(sh.tok[pos]) != 0);
    if (lane == 0) sh.tokb[row] = tb;
  }
  __syncthreads();
  if (tid < 32) {
    int tot = warp_prefix_words(sh.tokb, sh.tpref, S::NW, lane);
    if constexpr (MODEL == MODEL_BPE) {
      const int nl = sh.nl;
      if (nl) {  // (rare) word w also follows the tokens of the long pre-tokens that start in words before it
        for (int w = lane * 3; w < lane * 3 + 3 && w < S::NW; ++w) {
          int c = 0;
          for (int a = 0; a < nl; ++a) if (((int)sh.pt[sh.lk[a]] >> 5) < w) c = sh.lcum[a + 1];
          sh.tpref[w] += c;
        }
        tot += sh.lcum[nl];
      }
    }
    if (lane == 0) {
      sh.ntok = tot;
      P.tile_count[t] = (uint32_t)(tot + (sp.long_kept ? 1 : 0));
      P.tile_first[t] = (uint32_t)(base + sp.first);
    }
  }
}

// the page's tokens (long pre-tokens' included) before page position x < SPAN
template <class S>
__device__ __forceinline__ int tokens_before(const S& sh, int x) { return sh.tpref[x >> 5] + __popc(sh.tokb[x >> 5] & mask_lt(x & 31)); }

// P7: ids, offsets and word ids of the page's tokens at the provisional slots from base + first on.  A warp takes a word
// of tokb, a lane the token that starts at its position: its slot is the word's prefix plus its rank in the word.
template <int MODEL, unsigned LAY, class S>
__device__ __forceinline__ void emit_tokens(const ModelParams& P, const S& sh, int64_t base) {
  const PageSpan sp = page_span<MODEL>(sh);
  const unsigned long long excl = (unsigned long long)(base + sp.first);
  const int lane = threadIdx.x & 31;
  for (int row = threadIdx.x >> 5; row < S::NW; row += MODEL_THREADS / 32) {
    const uint32_t tb = sh.tokb[row];
    if (!((tb >> lane) & 1u)) continue;
    const int pos = row * 32 + lane;
    const uint32_t tk = sh.tok[pos];
    const int e = pos + tok_len(tk);
    emit_token<LAY>(P, sh, base, excl + (unsigned long long)(sh.tpref[row] + __popc(tb & mask_lt(lane))), tok_id(tk), pos,
                    bit_rank_incl(sh.lpref, sh.leadb, e - 1), base + e);
  }
  if constexpr (MODEL == MODEL_BPE) {
    // tokens of the long pre-tokens, produced by the pre-pass (positions relative to the pre-token start)
    for (int a = 0; a < sh.nl; ++a) {
      const int ls = sh.pt[sh.lk[a]];
      const int ntl = sh.lcum[a + 1] - sh.lcum[a];
      if (ntl == 0) continue;
      const uint4* __restrict__ lo = P.long_out + sh.loff[a];
      const unsigned long long obase = excl + (unsigned long long)tokens_before(sh, ls);
      const int X = bit_rank_incl(sh.lpref, sh.leadb, ls) - 1;  // chars of the page before the pre-token
      const DocOrigin o = doc_origin<LAY>(sh, base, ls);
      for (int k = threadIdx.x; k < ntl; k += MODEL_THREADS) {
        const uint4 r = lo[k];
        P.ids[obase + k] = r.x;
        place_token<LAY>(P, o, obase + k, X + (int)r.z, X + (int)r.w, base + ls + (k ? (int64_t)lo[k - 1].y : 0), base + ls + (int64_t)r.y);
      }
    }
  } else if (sp.long_kept && threadIdx.x == 0) {
    // chars up to the end of the long split = chars before it in the page + its own
    const int ls = sh.pt[sh.npt - 1];
    emit_token<LAY>(P, sh, base, excl + (unsigned long long)sh.ntok, P.t.unk_id, ls,
                    bit_rank_incl(sh.lpref, sh.leadb, ls) - 1 + sh.long_chars, sh.long_end);
  }
}

// P8: row_ptr of the documents starting in this page, page-local (row_ptr_fix_kernel adds the page's base)
template <class S>
__device__ __forceinline__ void write_row_ptr(const ModelParams& P, const S& sh, int64_t t, int64_t base) {
  const uint32_t fd = __ldg(P.page_first_doc + t);
  for (uint64_t d = (uint64_t)fd + threadIdx.x; d <= P.n_docs; d += MODEL_THREADS) {
    const int64_t pos = (int64_t)__ldg(P.doc_off + d) - base;
    if (pos >= TILE) break;
    // tokens that start before `pos` (a doc start is a pre-token start, so no token straddles it)
    P.row_ptr[d] = (unsigned long long)tokens_before(sh, (int)pos);
  }
}

constexpr int MODEL_MINBLOCKS = 8;  // 8 blocks/SM (32 regs, small spills) rather than 5 (48 regs): the kernel is latency-bound
template <int MODEL, unsigned LAY>
__global__ void __launch_bounds__(MODEL_THREADS, MODEL_MINBLOCKS) model_tile_kernel(const ModelParams P) {
  __shared__ __align__(16) PageState<MODEL> sh;
  const int tid = threadIdx.x;
  if (tid == 0) {
    sh.tile = (int)blockIdx.x;
    sh.nmiss = 0;
    if constexpr (MODEL == MODEL_BPE) { sh.nmiss_hi = 0; sh.nmq = 0; sh.anysoft = 0; sh.nl = 0; sh.lcum[0] = 0; }
    else { sh.next = 0; sh.long_chars = 0; }
  }
  __syncthreads();
  const int64_t t = sh.tile;
  if (t >= P.n_tiles) return;
  const int64_t base = t * TILE;

  stage_page<MODEL>(P, sh, t, base);
  __syncthreads();
  if constexpr (MODEL == MODEL_BPE) {
    collect_long_pretokens(P, sh, t, base);
    resolve_bpe(P, sh, t, base);
  } else {
    resolve_wordpiece(P, sh, t, base);
  }
  __syncthreads();
  count_tokens<MODEL>(P, sh, t, base);
  __syncthreads();
  emit_tokens<MODEL, LAY>(P, sh, base);
  write_row_ptr(P, sh, t, base);
}

// The instances of one model, in the order of MODEL_LAYOUTS
using ModelKernel = void (*)(const ModelParams);
template <int MODEL, int... I>
struct ModelKernelTable { static constexpr ModelKernel k[sizeof...(I)] = {&model_tile_kernel<MODEL, MODEL_LAYOUTS[I]>...}; };
template <int MODEL, int... I>
constexpr ModelKernelTable<MODEL, I...> model_kernel_table(std::integer_sequence<int, I...>) { return {}; }
template <int MODEL>
__host__ inline ModelKernel model_kernel(int layout_index) {
  using T = decltype(model_kernel_table<MODEL>(std::make_integer_sequence<int, N_MODEL_LAYOUTS>{}));
  return T::k[layout_index];
}


// ------------------------------------------------------------------------------------------------ pass 2
// Exclusive scan of the page token counts (two levels of 1024), then compaction of the provisional slots.
constexpr int TSCAN = 1024;

// exclusive scan of v over a block of TSCAN threads; s_w: 32 words of shared memory
__device__ __forceinline__ unsigned long long block_excl_scan(unsigned long long v, unsigned long long* s_w) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto warp_incl_scan = [lane](unsigned long long x) {
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) { unsigned long long o = __shfl_up_sync(0xFFFFFFFFu, x, s); if (lane >= s) x += o; }
    return x;
  };
  const unsigned long long inc = warp_incl_scan(v);
  if (lane == 31) s_w[warp] = inc;
  __syncthreads();
  if (warp == 0) { const unsigned long long w = s_w[lane]; s_w[lane] = warp_incl_scan(w) - w; }
  __syncthreads();
  return s_w[warp] + inc - v;
}

__global__ void __launch_bounds__(TSCAN) tile_scan_block_kernel(const uint32_t* __restrict__ cnt, unsigned long long* __restrict__ local_excl,
                                                                unsigned long long* __restrict__ block_sum, int64_t n_tiles) {
  __shared__ unsigned long long s_w[32];
  const int64_t i = (int64_t)blockIdx.x * TSCAN + threadIdx.x;
  const unsigned long long v = i < n_tiles ? (unsigned long long)cnt[i] : 0ull;
  const unsigned long long ex = block_excl_scan(v, s_w);
  if (i < n_tiles) local_excl[i] = ex;
  if (threadIdx.x == TSCAN - 1) block_sum[blockIdx.x] = ex + v;
}

__global__ void __launch_bounds__(TSCAN) tile_scan_top_kernel(unsigned long long* __restrict__ block_sum, int64_t n_blocks, unsigned long long* __restrict__ total) {
  __shared__ unsigned long long s_w[32];
  __shared__ unsigned long long s_run;
  if (threadIdx.x == 0) s_run = 0;
  __syncthreads();
  for (int64_t b0 = 0; b0 < n_blocks; b0 += TSCAN) {
    const int64_t i = b0 + threadIdx.x;
    const unsigned long long v = i < n_blocks ? block_sum[i] : 0ull;
    const unsigned long long ex = block_excl_scan(v, s_w);
    const unsigned long long run = s_run;
    if (i < n_blocks) block_sum[i] = run + ex;  // exclusive, in place
    __syncthreads();
    if (threadIdx.x == TSCAN - 1) s_run = run + ex + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = s_run;
}

// one warp per page: provisional slots -> final CSR positions.  A page has a few hundred tokens, so a warp copies only
// a dozen rounds of 32; each lane issues COMPACT_UNROLL rounds of loads before their stores, else every round waits for
// its loads and the copy is bound by memory latency rather than bandwidth.
constexpr int COMPACT_UNROLL = 8;
__global__ void compact_kernel(const uint32_t* __restrict__ tile_count, const uint32_t* __restrict__ tile_first,
                               const unsigned long long* __restrict__ local_excl, const unsigned long long* __restrict__ block_excl, int64_t n_tiles,
                               const uint32_t* __restrict__ t_ids, const uint2* __restrict__ t_off, const uint32_t* __restrict__ t_wid,
                               uint32_t* __restrict__ ids, uint2* __restrict__ off, uint32_t* __restrict__ wid) {
  const int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= n_tiles) return;
  const uint32_t cnt = tile_count[t];
  const unsigned long long src = tile_first[t], dst = local_excl[t] + block_excl[t / TSCAN];
  for (uint32_t j0 = lane; j0 < cnt; j0 += 32 * COMPACT_UNROLL) {
    uint32_t a[COMPACT_UNROLL], w[COMPACT_UNROLL];
    uint2 o[COMPACT_UNROLL];
#pragma unroll
    for (int u = 0; u < COMPACT_UNROLL; ++u) {
      const uint32_t j = j0 + 32 * u;
      if (j < cnt) {
        a[u] = t_ids[src + j];
        if (off) o[u] = t_off[src + j];
        if (wid) w[u] = t_wid[src + j];
      }
    }
#pragma unroll
    for (int u = 0; u < COMPACT_UNROLL; ++u) {
      const uint32_t j = j0 + 32 * u;
      if (j < cnt) {
        ids[dst + j] = a[u];
        if (off) off[dst + j] = o[u];
        if (wid) wid[dst + j] = w[u];
      }
    }
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
