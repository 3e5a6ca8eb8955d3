// encode_emul.cpp -- TEST ONLY: the encode path of the engine on the CPU.  The kernels of pretok_kernels.cuh,
// prefix_kernels.cuh, long_kernels.cuh and model_kernels.cuh are compiled unchanged behind simt.h (every thread a fiber,
// real warp semantics, several blocks at once) and run in engine.cu's order with its grid shapes:
//   [prefix re-pack] -> doc_mark -> K1 (the instance the engine picks) -> page_scan_block / page_scan_top ->
//   [BPE: long_find<0> -> soft_cut -> long_find<1> -> bpe_long] -> model_tile_kernel<MODEL, LAY> -> tile scans ->
//   compact -> row_ptr_fix
// on tables built by host_tables.cu (linked unchanged, as norm_emul does).  A few things the engine fixes are parameters:
// the SM count (it sizes the grids of K1, soft_cut and bpe_long), the word cache's slot count and whether it is on, the
// page kernel's output layout, and the seed that orders the lanes of a block.  Buffers the engine does not clear are
// filled with garbage first, outputs the layout does not write with a poison value.  The added-token extraction is not
// run here (tests/native/added_emul.cpp covers its kernels).
//   g++ -O2 -std=c++17 -I/usr/local/cuda/include -Wno-attributes -shared -fPIC -pthread -fvisibility=hidden -fno-gnu-unique \
//       -include cuda_runtime.h -o libencode_emul.so encode_emul.cpp -x c++ ../../tokenizers_b200/csrc/host_tables.cu
#include <cuda_runtime.h>
#include "simt.h"

#include <algorithm>
#include <string>
#include <vector>

// the word cache's fingerprint mask (b2t_emul_encode's Opts): 0 makes every fingerprint collide
static unsigned long long g_wc_fp_mask = ~0ull;
#define B2T_WC_TEST_FP_MASK g_wc_fp_mask

#include "../../include/b2t.h"
#include "../../tokenizers_b200/csrc/host_tables.h"
#include "../../tokenizers_b200/csrc/pretok_kernels.cuh"
#include "../../tokenizers_b200/csrc/prefix_kernels.cuh"
#include "../../tokenizers_b200/csrc/model_kernels.cuh"

using namespace b2t;

namespace {

constexpr uint32_t POISON = 0xDEADBEEFu;
constexpr uint8_t GARBAGE = 0xA5u;   // the bytes of workspace buffers the engine does not clear

struct Engine {
  int model = 0, pretok = 0, add_prefix_space = 0;
  HostTables ht;
  DeviceTables dt{};
};

// what one encode leaves behind, read by b2t_emul_get
struct Out {
  std::vector<uint32_t> ids, offsets, word_ids;   // final CSR (poison where the layout writes nothing)
  std::vector<uint64_t> row_ptr;
  std::vector<uint32_t> soft_bits;
  std::vector<LongDesc> desc1, desc;
  LongCtl lc{};
  uint32_t err = 0;
  uint64_t total = 0;
  uint64_t stray = 0;   // words of the provisional offsets / word ids the layout does not write that lost their poison
  int runs = 0;         // pipeline runs (a long pool that was too small makes the engine run the batch again)
  std::string error;
};
Out g_out;

template <class T>
void garbage(std::vector<T>& v, size_t n) { v.assign(n, T()); memset(v.data(), GARBAGE, n * sizeof(T)); }

struct Opts {
  uint32_t layout;        // an entry of MODEL_LAYOUTS
  uint32_t wcache_slots;  // power of two
  int32_t wcache_on;
  int32_t sm_count;
  uint64_t seed;          // 0: lanes in thread order
  uint64_t wc_fp_mask;    // word-cache fingerprints & this (the product keeps all 62 bits)
};

#define LAUNCH(name, grid, block, ...)                                                              \
  do {                                                                                              \
    std::string e_ = simt::launch(name, dim3(grid), dim3(block), o.seed, [&] { __VA_ARGS__; });     \
    if (!e_.empty()) { g_out.error = e_; return 1; }                                                \
  } while (0)

template <int KIND>
int launch_k1(const Opts& o, const uint8_t* bytes, int64_t n, const uint32_t* doc_bits, const uint32_t* cls, uint32_t* start_bits,
              uint32_t* drop_bits, uint64_t* page_sum) {
  // launch_pretok of engine.cu
  const int64_t n_chunks = n / CHUNK + 1;
  const int64_t n_kb = (n_chunks + 31) / 32;
  const int64_t resident = (int64_t)o.sm_count * (KIND == PT_LLAMA3 ? K1_WINDOW_MINBLOCKS : K1_LEAN_MINBLOCKS) * (K1_THREADS / 32);
  int64_t kb = (n_kb + resident * 4 - 1) / (resident * 4);
  kb = std::min<int64_t>(128, std::max<int64_t>(2, (kb + 1) & ~1ll));
  const int64_t n_warps = (n_kb + kb - 1) / kb;
  const unsigned grid = (unsigned)((n_warps + (K1_THREADS / 32) - 1) / (K1_THREADS / 32));
  if constexpr (KIND == PT_LLAMA3) {
    LAUNCH("pretok_stream_kernel", grid, K1_THREADS, pretok_stream_kernel<KIND>(bytes, n, doc_bits, cls, start_bits, page_sum, (int)n_kb, (int)kb));
  } else {
    const SwapMasks masks{0x55555555u, 0x33333333u, 0x0F0F0F0Fu};
    LAUNCH("pretok_lean_kernel", grid, K1_THREADS, pretok_lean_kernel<KIND>(bytes, n, doc_bits, cls, start_bits, drop_bits, page_sum, (int)n_kb, (int)kb, masks));
  }
  return 0;
}

// one run of the pipeline on the (re-packed) batch; pool_cap: bytes of long pre-tokens the long pool holds
int run(const Engine& E, const Opts& o, const uint8_t* bytes, int64_t n, const uint64_t* doc_off, uint32_t n_docs,
        const uint32_t* prefix_bits, unsigned long long pool_cap) {
  const bool bpe = E.model == MODEL_BPE;
  const int64_t n_words = n / 32 + 2, n_pages = n / PAGE + 1;
  const unsigned lay = o.layout;
  // size_buffers: cleared as the engine clears them, the rest holds garbage
  std::vector<uint32_t> doc_bits(n_words, 0u), start_bits, drop_bits, page_first_doc;
  std::vector<uint64_t> page_sum, page_carry, block_sum, block_carry;
  garbage(start_bits, n_words); garbage(drop_bits, n_words); garbage(page_first_doc, n_pages);
  garbage(page_sum, n_pages); garbage(page_carry, n_pages);
  garbage(block_sum, n_pages / SCAN_BLOCK + 2); garbage(block_carry, n_pages / SCAN_BLOCK + 2);
  struct { LongCtl lc; unsigned long long total; uint32_t err; } ctl{};
  std::vector<uint4> wcache((size_t)o.wcache_slots * 4, make_uint4(0u, 0u, 0u, 0u));
  std::vector<uint32_t> soft_bits(n_words, 0u);
  std::vector<uint8_t> page_soft(n_pages, 0u);
  std::vector<int32_t> page_long;
  std::vector<LongDesc> long_desc, long_desc1;
  garbage(page_long, n_pages);
  garbage(long_desc, (size_t)(n / (LONG_PRETOK_MIN + 1) + 2)); garbage(long_desc1, (size_t)(n / (LONG_PRETOK_MIN + 1) + 2));
  std::vector<uint32_t> lp_id, lp_len, lp_plen, lp_aux;
  std::vector<uint64_t> lp_val;
  std::vector<uint4> lp_out;
  garbage(lp_id, pool_cap); garbage(lp_len, pool_cap); garbage(lp_plen, pool_cap); garbage(lp_aux, pool_cap); garbage(lp_val, pool_cap);
  garbage(lp_out, pool_cap);
  std::vector<uint32_t> tmp_ids, tmp_off, tmp_wid, tile_count, tile_first;
  std::vector<uint64_t> row_ptr_local;
  std::vector<unsigned long long> tile_lexcl, tile_bsum;
  garbage(tmp_ids, n + 1); tmp_off.assign((size_t)(n + 1) * 2, POISON); tmp_wid.assign(n + 1, POISON);
  garbage(tile_count, n_pages); garbage(tile_first, n_pages); garbage(row_ptr_local, (size_t)n_docs + 1);
  garbage(tile_lexcl, n_pages); garbage(tile_bsum, n_pages / TSCAN + 2);
  Out& r = g_out;
  r.ids.assign(n + 1, POISON); r.offsets.assign((size_t)(n + 1) * 2, POISON); r.word_ids.assign(n + 1, POISON);
  r.row_ptr.assign((size_t)n_docs + 1, 0ull);
  memset(r.row_ptr.data(), GARBAGE, r.row_ptr.size() * 8);

  // K0, K1, K1b
  LAUNCH("doc_mark_kernel", (n_docs + 1 + 255) / 256, 256, doc_mark_kernel(doc_off, n_docs, doc_bits.data(), page_first_doc.data()));
  const uint32_t* cls = E.ht.cls_packed.data();
  int rc = 0;
  switch (E.pretok) {
    case PT_GPT2: rc = launch_k1<PT_GPT2>(o, bytes, n, doc_bits.data(), cls, start_bits.data(), drop_bits.data(), page_sum.data()); break;
    case PT_LLAMA3: rc = launch_k1<PT_LLAMA3>(o, bytes, n, doc_bits.data(), cls, start_bits.data(), drop_bits.data(), page_sum.data()); break;
    case PT_WHITESPACE: rc = launch_k1<PT_WHITESPACE>(o, bytes, n, doc_bits.data(), cls, start_bits.data(), drop_bits.data(), page_sum.data()); break;
    case PT_BERT: rc = launch_k1<PT_BERT>(o, bytes, n, doc_bits.data(), cls, start_bits.data(), drop_bits.data(), page_sum.data()); break;
    default: rc = launch_k1<PT_NOREGEX>(o, bytes, n, doc_bits.data(), cls, start_bits.data(), drop_bits.data(), page_sum.data()); break;
  }
  if (rc) return rc;
  const int64_t n_scan_blocks = (n_pages + SCAN_BLOCK - 1) / SCAN_BLOCK;
  LAUNCH("page_scan_block_kernel", (unsigned)n_scan_blocks, SCAN_BLOCK, page_scan_block_kernel(page_sum.data(), page_carry.data(), block_sum.data(), n_pages));
  LAUNCH("page_scan_top_kernel", 1, SCAN_BLOCK, page_scan_top_kernel(block_sum.data(), block_carry.data(), n_scan_blocks));

  // K1c / K2L
  LongPool pool;
  pool.id = lp_id.data(); pool.val = lp_val.data(); pool.len = lp_len.data(); pool.plen = lp_plen.data(); pool.aux = lp_aux.data();
  pool.out = lp_out.data(); pool.cap = pool_cap;
  if (bpe) {
    LAUNCH("long_find_kernel<0>", (unsigned)((n_pages + 7) / 8), 256,
           long_find_kernel<0>(start_bits.data(), nullptr, nullptr, n, n_pages, &ctl.lc, long_desc1.data(), nullptr, 0ull));
    LAUNCH("soft_cut_kernel", (unsigned)(o.sm_count * 4), 256, soft_cut_kernel(bytes, &ctl.lc, long_desc1.data(), soft_bits.data(), page_soft.data(), E.dt));
    LAUNCH("long_find_kernel<1>", (unsigned)((n_pages + 7) / 8), 256,
           long_find_kernel<1>(start_bits.data(), soft_bits.data(), page_soft.data(), n, n_pages, &ctl.lc, long_desc.data(), page_long.data(), pool_cap));
    LAUNCH("bpe_long_kernel", (unsigned)(o.sm_count * 2), LONG_THREADS, bpe_long_kernel(bytes, &ctl.lc, long_desc.data(), pool, E.dt, E.dt.monotone));
  }

  // K2
  ModelParams P;
  memset(&P, 0, sizeof(P));
  P.bytes = bytes; P.n = n;
  P.start_bits = start_bits.data(); P.drop_bits = drop_bits.data(); P.doc_bits = doc_bits.data();
  P.soft_bits = soft_bits.data(); P.page_soft = page_soft.data();
  P.page_carry = page_carry.data(); P.block_carry = block_carry.data(); P.page_first_doc = page_first_doc.data();
  P.doc_off = doc_off; P.n_docs = n_docs;
  P.ids = tmp_ids.data(); P.offsets = tmp_off.data(); P.word_ids = tmp_wid.data(); P.row_ptr = row_ptr_local.data();
  P.tile_count = tile_count.data(); P.tile_first = tile_first.data(); P.err_flag = &ctl.err; P.n_tiles = n_pages;
  P.page_long = page_long.data(); P.long_desc = long_desc.data(); P.long_out = lp_out.data();
  P.wcache = wcache.data(); P.wcache_mask = o.wcache_slots - 1; P.wcache_on = o.wcache_on;
  P.prefix_bits = prefix_bits;
  P.added_bits = nullptr; P.added_head = nullptr; P.added_pool = nullptr;
  P.t = E.dt;
  const int li = model_layout_index(lay);
  const ModelKernel k = bpe ? model_kernel<MODEL_BPE>(li) : model_kernel<MODEL_WORDPIECE>(li);
  const std::string kname = std::string("model_tile_kernel<") + (bpe ? "MODEL_BPE" : "MODEL_WORDPIECE") + ", " + std::to_string(lay) + ">";
  LAUNCH(kname.c_str(), (unsigned)n_pages, MODEL_THREADS, k(P));
  const int64_t n_tblk = (n_pages + TSCAN - 1) / TSCAN;
  LAUNCH("tile_scan_block_kernel", (unsigned)n_tblk, TSCAN, tile_scan_block_kernel(tile_count.data(), tile_lexcl.data(), tile_bsum.data(), n_pages));
  LAUNCH("tile_scan_top_kernel", 1, TSCAN, tile_scan_top_kernel(tile_bsum.data(), n_tblk, &ctl.total));

  // pass 2 (finish_device): outputs the layout does not want are not passed
  const bool offs = lay & L_OFFSETS, wids = lay & L_WORD_IDS;
  LAUNCH("compact_kernel", (unsigned)((n_pages * 32 + 255) / 256), 256,
         compact_kernel(tile_count.data(), tile_first.data(), tile_lexcl.data(), tile_bsum.data(), n_pages, tmp_ids.data(),
                        offs ? reinterpret_cast<const uint2*>(tmp_off.data()) : nullptr, wids ? tmp_wid.data() : nullptr, r.ids.data(),
                        offs ? reinterpret_cast<uint2*>(r.offsets.data()) : nullptr, wids ? r.word_ids.data() : nullptr));
  LAUNCH("row_ptr_fix_kernel", (n_docs + 1 + 255) / 256, 256,
         row_ptr_fix_kernel(doc_off, n_docs, tile_lexcl.data(), tile_bsum.data(), row_ptr_local.data(), r.row_ptr.data(), 0ull));

  r.stray = 0;
  if (!offs) for (uint32_t v : tmp_off) r.stray += v != POISON;
  if (!wids) for (uint32_t v : tmp_wid) r.stray += v != POISON;
  r.soft_bits.assign(soft_bits.begin(), soft_bits.begin() + (n / 32 + 1));
  r.lc = ctl.lc;
  r.desc1.assign(long_desc1.begin(), long_desc1.begin() + (bpe ? std::min<size_t>(ctl.lc.n_long1, long_desc1.size()) : 0));
  r.desc.assign(long_desc.begin(), long_desc.begin() + (bpe ? std::min<size_t>(ctl.lc.n_long, long_desc.size()) : 0));
  r.err = ctl.err | ctl.lc.err;
  r.total = ctl.total;
  return 0;
}

}  // namespace

// Only the b2t_emul_* entry points leave the library (it is built with -fvisibility=hidden -fno-gnu-unique): the kernels,
// their instance tables and host_tables.cu are also in the engine's library, under the same names, and a process that
// loads both must keep each library bound to its own copies.
#pragma GCC visibility push(default)
extern "C" {

// The tables of a b2t_config as b2t_engine_create builds them; NULL on error (message in err).
void* b2t_emul_create(const b2t_config* cfg, char* err, int err_len) {
  Engine* E = new Engine();
  bool vocab_err = false;
  const std::string msg = build_host_tables(cfg->model, cfg->pretok, cfg->ignore_merges, cfg->n_vocab, cfg->vocab_bytes, cfg->vocab_off, cfg->vocab_ids,
                                            cfg->n_merges, cfg->merge_bytes, cfg->merge_off, cfg->unk_token, cfg->continuing_subword_prefix,
                                            cfg->max_input_chars_per_word, &E->ht, &vocab_err);
  if (!msg.empty()) { snprintf(err, err_len, "%s", msg.c_str()); delete E; return nullptr; }
  E->model = cfg->model; E->pretok = cfg->pretok; E->add_prefix_space = cfg->add_prefix_space;
  const HostTables& ht = E->ht;
  DeviceTables& t = E->dt;
  t.byte_to_id = ht.byte_to_id.data();
  t.merge_tbl = ht.merge_tbl.data(); t.merge_mask = ht.merge_tbl.empty() ? 0 : (uint32_t)ht.merge_tbl.size() - 1;
  t.word_tbl = ht.word_tbl.data(); t.word_mask = ht.word_tbl.empty() ? 0 : (uint32_t)ht.word_tbl.size() - 1;
  t.word_pool = ht.word_pool.data();
  t.ignore_merges = cfg->ignore_merges ? 1 : 0;
  t.monotone = ht.monotone ? 1 : 0;
  t.tok2_bits = ht.tok2_bits.data(); t.tri_bits = ht.tri_bits.data();
  t.edge_tbl = ht.edge_tbl.data(); t.edge_mask = ht.edge_tbl.empty() ? 0 : (uint32_t)ht.edge_tbl.size() - 1;
  t.unk_id = ht.unk_id; t.max_chars = ht.max_chars;
  return E;
}
void b2t_emul_destroy(void* e) { delete static_cast<Engine*>(e); }
int b2t_emul_monotone(void* e) { return static_cast<Engine*>(e)->ht.monotone ? 1 : 0; }

// Encodes a packed batch; 0 = done (read the outputs with b2t_emul_get), 1 = a check of the SIMT runtime failed (message
// from b2t_emul_error), 2 = the layout does not exist.  Like check_run, a long pool that was too small is grown to what
// the run asked for and the batch runs again.
int b2t_emul_encode(void* eh, const uint8_t* bytes, int64_t n, const uint64_t* doc_off, uint32_t n_docs, const Opts* opt) {
  const Engine& E = *static_cast<Engine*>(eh);
  const Opts& o = *opt;
  g_out = Out();
  if (model_layout_index(o.layout) < 0) return 2;
  g_wc_fp_mask = o.wc_fp_mask;
  // repack_prefix
  std::vector<uint8_t> pfx_bytes;
  std::vector<uint64_t> pfx_off;
  std::vector<uint32_t> prefix_bits;
  const uint32_t* pbits = nullptr;
  if (E.add_prefix_space && n_docs && n) {
    const int64_t cap = n + n_docs + 64;
    const uint32_t nb = (n_docs + PFX_BLOCK - 1) / PFX_BLOCK;
    pfx_bytes.assign(cap, GARBAGE); garbage(pfx_off, (size_t)n_docs + 1);
    prefix_bits.assign(cap / 32 + 2, 0u);
    std::vector<uint32_t> local, block;
    garbage(local, n_docs); garbage(block, nb + 4);
    unsigned long long total = 0;
    LAUNCH("pfx_scan_block_kernel", nb, PFX_BLOCK, pfx_scan_block_kernel(bytes, doc_off, n_docs, local.data(), block.data()));
    LAUNCH("pfx_scan_top_kernel", 1, PFX_BLOCK, pfx_scan_top_kernel(block.data(), nb, &total));
    LAUNCH("pfx_offsets_kernel", (n_docs + 1 + 255) / 256, 256,
           pfx_offsets_kernel(bytes, doc_off, n_docs, local.data(), block.data(), &total, pfx_off.data(), prefix_bits.data()));
    LAUNCH("pfx_copy_kernel", (unsigned)(((int64_t)n_docs * 32 + 255) / 256), 256, pfx_copy_kernel(bytes, doc_off, pfx_off.data(), n_docs, pfx_bytes.data()));
    bytes = pfx_bytes.data(); doc_off = pfx_off.data(); n += (int64_t)total;
    pbits = prefix_bits.data();
  } else if (o.layout & L_PREFIX) {
    // the instance exists for every model: without a prefix pipeline it reads a bitmap without prefix spaces
    prefix_bits.assign(n / 32 + 2, 0u);
    pbits = prefix_bits.data();
  }
  unsigned long long cap = (1u << 20) + (1u << 20) / 4 + 4096;   // ensure_long_pool(1 << 20)
  for (int attempt = 0;; ++attempt) {
    g_out.runs = attempt + 1;
    if (run(E, o, bytes, n, doc_off, n_docs, pbits, cap)) return 1;
    if (!(g_out.lc.err & ERR_POOL_OVERFLOW) || attempt >= 2) break;
    const unsigned long long want = g_out.lc.pool_used;
    cap = want + want / 4 + 4096;
  }
  return 0;
}

const char* b2t_emul_error() { return g_out.error.c_str(); }

// sizes of the outputs: tokens, long descriptors of the first and the second pass, soft-bit words
void b2t_emul_sizes(uint64_t* out) {
  out[0] = g_out.total; out[1] = g_out.desc1.size(); out[2] = g_out.desc.size(); out[3] = g_out.soft_bits.size();
  out[4] = g_out.err; out[5] = g_out.stray; out[6] = g_out.runs;
  out[7] = g_out.lc.n_long1; out[8] = g_out.lc.n_long; out[9] = g_out.lc.pool_used;
}

// ids[T], offsets[2T], word_ids[T], row_ptr[n_docs + 1], soft_bits[words]; desc: {start, end, pool_off, ntok | soft << 32}
// per descriptor (first pass, then second pass)
void b2t_emul_get(uint32_t* ids, uint32_t* offsets, uint32_t* word_ids, uint64_t* row_ptr, uint32_t* soft_bits, uint64_t* desc1, uint64_t* desc) {
  const size_t T = g_out.total;
  memcpy(ids, g_out.ids.data(), T * 4);
  memcpy(offsets, g_out.offsets.data(), T * 8);
  memcpy(word_ids, g_out.word_ids.data(), T * 4);
  memcpy(row_ptr, g_out.row_ptr.data(), g_out.row_ptr.size() * 8);
  memcpy(soft_bits, g_out.soft_bits.data(), g_out.soft_bits.size() * 4);
  auto put = [](const std::vector<LongDesc>& v, uint64_t* d) {
    for (size_t i = 0; i < v.size(); ++i) {
      d[4 * i] = (uint64_t)v[i].start; d[4 * i + 1] = (uint64_t)v[i].end; d[4 * i + 2] = v[i].pool_off;
      d[4 * i + 3] = v[i].ntok | ((uint64_t)v[i].soft << 32);
    }
  };
  put(g_out.desc1, desc1);
  put(g_out.desc, desc);
}

// every entry of MODEL_LAYOUTS
int b2t_emul_layouts(uint32_t* out) {
  for (int i = 0; i < N_MODEL_LAYOUTS; ++i) out[i] = MODEL_LAYOUTS[i];
  return N_MODEL_LAYOUTS;
}

}  // extern "C"
#pragma GCC visibility pop
