// engine.cu -- the C ABI of include/b2t.h: engine construction, the device pipeline ([N1-N2 BertNormalizer pre-pass ->]
// K0 doc_mark -> [A1-A2 added-token extraction ->] K1 pretok_scan -> K1b page_scan -> [K1c / K2L long pre-tokens ->]
// K2 model_tile -> K2b scan + compaction [-> N3 offsets back to the original text] [-> dense rows]) and the chunked
// host<->device pipeline of b2t_encode_batch / b2t_encode_batch_dense.
//
// This is the batch-level seam of the reference (tokenizer/mod.rs:1337-1401 encode_batch*): one call = one batch,
// results in input order, any failure fails the whole batch.  There is NO CPU implementation behind these entry
// points; without a CUDA device they fail with B2T_ERR_CUDA.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b2t.h"
#include "added_kernels.cuh"
#include "dense_kernels.cuh"
#include "host_tables.h"
#include "long_kernels.cuh"
#include "model_kernels.cuh"
#include "norm_kernels.cuh"
#include "prefix_kernels.cuh"
#include "pretok_kernels.cuh"

using namespace b2t;

// ------------------------------------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define CU(call)                                                                                              \
  do {                                                                                                        \
    cudaError_t _e = (call);                                                                                  \
    if (_e != cudaSuccess) return fail(B2T_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

extern "C" const char* b2t_last_error(void) { return g_err; }
extern "C" const char* b2t_version(void) { return "tokenizers_b200 0.1 (sm_90a)"; }

extern "C" int b2t_bert_normalizer_images(int32_t flags, uint8_t* pool, size_t cap, uint32_t* off) {
  if (!pool || !off) return fail(B2T_ERR_INVALID, "b2t_bert_normalizer_images: null argument");
  NormHost nh;
  build_bert_norm((flags & B2T_NORM_CLEAN_TEXT) != 0, (flags & B2T_NORM_CHINESE_CHARS) != 0, (flags & B2T_NORM_STRIP_ACCENTS) != 0, (flags & B2T_NORM_LOWERCASE) != 0, &nh);
  size_t pos = 0;
  for (uint32_t c = 0; c < 0x110000; ++c) {
    off[c] = (uint32_t)pos;
    const uint32_t e = nh.ent[(size_t)nh.blk[c >> 7] * 128 + (c & 127)], kind = e & 3u;
    if (kind == NORM_REMOVE || (c >= 0xD800 && c <= 0xDFFF)) continue;
    uint8_t tmp[4]; const uint8_t* src = tmp; size_t len;
    if (kind == NORM_STRING) { src = nh.pool.data() + (e >> 8); len = (e >> 2) & 63u; }
    else {   // the character itself
      if (c < 0x80) { tmp[0] = (uint8_t)c; len = 1; }
      else if (c < 0x800) { tmp[0] = 0xC0 | (c >> 6); tmp[1] = 0x80 | (c & 63); len = 2; }
      else if (c < 0x10000) { tmp[0] = 0xE0 | (c >> 12); tmp[1] = 0x80 | ((c >> 6) & 63); tmp[2] = 0x80 | (c & 63); len = 3; }
      else { tmp[0] = 0xF0 | (c >> 18); tmp[1] = 0x80 | ((c >> 12) & 63); tmp[2] = 0x80 | ((c >> 6) & 63); tmp[3] = 0x80 | (c & 63); len = 4; }
    }
    if (pos + len > cap) return fail(B2T_ERR_TOO_LARGE, "b2t_bert_normalizer_images: pool too small");
    memcpy(pool + pos, src, len);
    pos += len;
  }
  off[0x110000] = (uint32_t)pos;
  return B2T_OK;
}

extern "C" int b2t_unicode_class_table(int scheme, uint8_t* out) {
  if (!out || (scheme != 0 && scheme != 1 && scheme != 2)) return fail(B2T_ERR_INVALID, "b2t_unicode_class_table: bad arguments");
  unicode_class_table(scheme, out);
  return B2T_OK;
}

// ------------------------------------------------------------------------------------------------ buffers
// Device and pinned host buffers own their memory: it is freed with the buffer (after the owner has synchronised).  They
// are move-only: declaring the move constructor deletes the copies.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  ~DevBuf() { if (p) cudaFree(p); }
  int ensure(size_t bytes) {
    if (bytes <= cap) return B2T_OK;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    CU(cudaMalloc(&p, want));
    cap = want;
    return B2T_OK;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};
struct PinBuf {
  void* p = nullptr;
  size_t cap = 0;
  PinBuf() = default;
  PinBuf(PinBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  ~PinBuf() { if (p) cudaFreeHost(p); }
  int ensure(size_t bytes, bool keep) {
    if (bytes <= cap) return B2T_OK;
    size_t want = bytes + bytes / 4 + 4096;
    void* q = nullptr;
    CU(cudaHostAlloc(&q, want, cudaHostAllocDefault));
    if (p) { if (keep) memcpy(q, p, cap); cudaFreeHost(p); }
    p = q; cap = want;
    return B2T_OK;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

// Dense mode request (b2t_encode_batch_dense*): the device-side spec plus how L is chosen.
struct DenseReq {
  DenseSpec S;
  bool batch_longest = false;   // padding strategy BatchLongest: L = longest row of the batch (after pad_to_multiple_of)
  uint32_t multiple = 0;        // pad_to_multiple_of
  bool want_mask = false;
};

// How far run_device_pipeline goes: pre-tokenization only (K0..K1b), up to the token count (the caller finishes into its
// own buffers), or the whole result in the workspace.
enum RunUntil { RUN_PRETOK, RUN_COUNT, RUN_RESULT };

// The inputs of one pipeline run, kept so that the run can be repeated with a larger long pool.  `dq` (dense mode) points
// at the caller's request and is only valid during the call.
struct Request {
  const uint8_t* bytes = nullptr; int64_t n = 0; const uint64_t* doc_off = nullptr; uint32_t n_docs = 0, flags = 0;
  RunUntil until = RUN_RESULT; const DenseReq* dq = nullptr;
};

// The batch the kernels ran on: the request's, or its re-packed (add_prefix_space) or normalized copy in the workspace.
struct Batch {
  const uint8_t* bytes = nullptr; int64_t n = 0; const uint64_t* doc_off = nullptr; uint32_t n_docs = 0;
  const uint32_t* prefix_bits = nullptr;
};

// Device-side state of one in-flight batch (or chunk).
struct Workspace {
  DevBuf bytes, doc_off;              // only used by the host path (inputs staged on the device)
  DevBuf doc_bits, start_bits, drop_bits, page_sum, page_carry, block_sum, block_carry, page_first_doc, ctl;
  DevBuf ids, offsets, word_ids, row_ptr, row_ptr_local;
  Request req;                        // the last run
  Batch batch;
  bool pending = false;               // begin / finish
  DevBuf tmp_ids, tmp_offsets, tmp_word_ids, tile_count, tile_first, tile_lexcl, tile_bsum;  // pass-1 provisional slots + scan
  DevBuf page_long, long_desc, long_desc1, soft_bits, page_soft, lp_id, lp_val, lp_len, lp_plen, lp_aux, lp_out;  // long BPE pre-tokens (long_kernels.cuh)
  unsigned long long pool_cap = 0;
  DevBuf wcache;                      // per-batch word cache (model_kernels.cuh)
  DevBuf dense_ids, dense_mask, dense_len;  // dense [n_docs, L] rows (dense_kernels.cuh)
  // BertNormalizer pre-pass (norm_kernels.cuh): the normalized batch and what maps its tokens back to the original
  DevBuf nrm_doc_bits, nrm_pfd, nrm_page_out, nrm_page_chars, nrm_lexcl_o, nrm_bsum_o, nrm_lexcl_c, nrm_bsum_c, nrm_tot, nrm_bytes, nrm_src_char, nrm_doc_off, nrm_doc_char0;
  bool norm_active = false;
  DevBuf cand0, cand1, cand_any, hard_bits, inner_bits, added_bits, added_head, added_pool;
  uint32_t added_cap = 0;  // added-token extraction (added_kernels.cuh)
  DevBuf pfx_bytes, pfx_doc_off, pfx_local, pfx_block, prefix_bits, pfx_total;  // add_prefix_space re-pack (prefix_kernels.cuh)
  cudaStream_t stream = nullptr;
  cudaEvent_t done = nullptr;
  PinBuf h_ctl;                        // total tokens + error flag read back
  ~Workspace() {                       // (not copyable: the buffers are not)
    if (stream) cudaStreamDestroy(stream);
    if (done) cudaEventDestroy(done);
  }
};

struct b2t_result {
  b2t_engine* eng = nullptr;
  int on_device = 0;
  uint32_t n_docs = 0;
  uint64_t n_tokens = 0;
  const uint32_t* ids = nullptr; const uint32_t* offsets = nullptr; const uint32_t* word_ids = nullptr; const uint64_t* row_ptr = nullptr;
  PinBuf h_ids, h_offsets, h_word_ids, h_row_ptr;  // host results own pinned memory (returned to the engine pool on free)
  // dense mode (b2t_encode_batch_dense*): [n_docs, dense_len] rows instead of the CSR
  uint32_t dense_len = 0;
  const uint32_t* dense_ids = nullptr; const uint8_t* dense_mask = nullptr; const uint32_t* row_len = nullptr;
  PinBuf h_dense_ids, h_dense_mask, h_row_len;
};

constexpr int NSLOT = 3;   // chunk workspaces of one host-path call: NSLOT - 1 chunks are in flight while the next is issued
constexpr int MAX_KERNEL_RECORDS = 16;

struct b2t_engine {
  int device = 0;
  int model = 0, pretok = 0, add_prefix_space = 0;
  int sm_count = 132;
  int wcache_on = 1;         // B2T_WCACHE=0: no word cache, every pre-token is merged (the reference benches cache_capacity(0) too)
  DeviceTables dt;
  int monotone = 0;
  DevBuf d_cls, d_byte_to_id, d_merge, d_word, d_pool, d_edge, d_tok2, d_tri;
  // BertNormalizer (b2t_config.bert_normalizer)
  int norm_on = 0;
  NormTables nt;
  DevBuf d_nt_blk, d_nt_ent, d_nt_pool, d_nt_ascii;
  // added vocabulary (b2t_engine_set_added_tokens)
  int has_added = 0;
  AddedTables at;
  DevBuf d_at_bytes, d_at_off, d_at_id, d_at_flags, d_at_first, d_at_pair, d_cls_rust;
  // Concurrency: the tables are immutable, every host-path call (b2t_encode_batch, _dense, b2t_pre_tokenize_batch) runs on a
  // slot set of its own -- NSLOT workspaces with their streams -- so calls from several host threads overlap their copies
  // and kernels; `mu` only guards the pools (and the whole call while per-kernel profiling is on: the event records are one
  // per engine).  The device-resident entry points keep one workspace (their result lives in it) and serialise on `mu`.
  std::mutex mu;        // pools of results and slot sets (held briefly)
  std::mutex dev_mu;    // the device-resident entry points, whole call
  std::mutex prof_mu;   // host-path calls while profiling is on, whole call
  std::condition_variable set_free;
  Workspace dev_ws;          // b2t_encode_batch_device
  struct SlotSet { Workspace slot[NSLOT]; bool busy = false; };
  std::vector<std::unique_ptr<SlotSet>> sets;   // at most MAX_SLOT_SETS, created on demand
  cudaStream_t own_stream = nullptr;
  size_t chunk_bytes = 64u << 20;
  // pinned result pool
  std::vector<std::unique_ptr<b2t_result>> pool;
  // profiling
  int profiling = 0;
  int n_rec = 0;
  const char* rec_name[MAX_KERNEL_RECORDS];
  cudaEvent_t rec_ev[MAX_KERNEL_RECORDS + 1];
  bool rec_ev_made = false;
  std::atomic<int> last_launches{0};
  ~b2t_engine() {   // (b2t_engine_destroy has set the device and synchronised; the buffers free themselves after this)
    if (rec_ev_made) for (auto& ev : rec_ev) cudaEventDestroy(ev);
    if (own_stream) cudaStreamDestroy(own_stream);
  }
};
constexpr size_t MAX_SLOT_SETS = 4;

// ------------------------------------------------------------------------------------------------ create / destroy
template <class T>
static int upload(DevBuf& b, const std::vector<T>& v) {
  size_t bytes = v.size() * sizeof(T);
  int rc = b.ensure(bytes ? bytes : 16);
  if (rc) return rc;
  if (bytes) CU(cudaMemcpy(b.p, v.data(), bytes, cudaMemcpyHostToDevice));
  return B2T_OK;
}

extern "C" int b2t_engine_create(const b2t_config* cfg, b2t_engine** out) {
  if (!cfg || !out) return fail(B2T_ERR_INVALID, "b2t_engine_create: null argument");
  if (cfg->struct_size != sizeof(b2t_config)) return fail(B2T_ERR_INVALID, "b2t_engine_create: struct_size mismatch (%u != %zu)", cfg->struct_size, sizeof(b2t_config));
  *out = nullptr;
  if (cfg->model != B2T_MODEL_BPE && cfg->model != B2T_MODEL_WORDPIECE) return fail(B2T_ERR_UNSUPPORTED, "unsupported model kind %d", cfg->model);
  if (cfg->pretok < 0 || cfg->pretok > 4) return fail(B2T_ERR_UNSUPPORTED, "unsupported pre-tokenizer kind %d", cfg->pretok);
  if (cfg->model == B2T_MODEL_BPE && (cfg->pretok == B2T_PRETOK_WHITESPACE || cfg->pretok == B2T_PRETOK_BERT))
    return fail(B2T_ERR_UNSUPPORTED, "BPE is supported behind the ByteLevel pre-tokenizers only");
  if (cfg->model == B2T_MODEL_WORDPIECE && cfg->pretok != B2T_PRETOK_WHITESPACE && cfg->pretok != B2T_PRETOK_BERT)
    return fail(B2T_ERR_UNSUPPORTED, "WordPiece is supported behind the Whitespace and Bert pre-tokenizers only");
  if ((cfg->bert_normalizer & B2T_NORM_BERT) && cfg->model != B2T_MODEL_WORDPIECE)
    return fail(B2T_ERR_UNSUPPORTED, "BertNormalizer is supported in front of WordPiece pipelines only");
  if (cfg->bert_normalizer & ~(B2T_NORM_BERT | B2T_NORM_CLEAN_TEXT | B2T_NORM_CHINESE_CHARS | B2T_NORM_STRIP_ACCENTS | B2T_NORM_LOWERCASE))
    return fail(B2T_ERR_INVALID, "unknown bits in bert_normalizer");
  if (cfg->add_prefix_space && cfg->pretok != B2T_PRETOK_BYTELEVEL && cfg->pretok != B2T_PRETOK_BYTELEVEL_NOREGEX)
    return fail(B2T_ERR_UNSUPPORTED, "add_prefix_space is only meaningful for a top-level ByteLevel pre-tokenizer");
  if (!cfg->vocab_bytes || !cfg->vocab_off || !cfg->vocab_ids || cfg->n_vocab == 0) return fail(B2T_ERR_INVALID, "empty vocabulary");

  HostTables ht;
  bool vocab_err = false;
  std::string msg = build_host_tables(cfg->model, cfg->pretok, cfg->ignore_merges, cfg->n_vocab, cfg->vocab_bytes, cfg->vocab_off,
                                      cfg->vocab_ids, cfg->n_merges, cfg->merge_bytes, cfg->merge_off, cfg->unk_token,
                                      cfg->continuing_subword_prefix, cfg->max_input_chars_per_word, &ht, &vocab_err);
  if (!msg.empty()) return fail(vocab_err ? B2T_ERR_VOCAB : B2T_ERR_UNSUPPORTED, "%s", msg.c_str());

  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return fail(B2T_ERR_CUDA, "no CUDA device available (%s); this engine has no CPU path", cudaGetErrorString(ce));
  int dev = cfg->device;
  if (dev < 0) CU(cudaGetDevice(&dev));
  if (dev >= ndev) return fail(B2T_ERR_INVALID, "device %d out of range (%d devices)", dev, ndev);
  CU(cudaSetDevice(dev));

  std::unique_ptr<b2t_engine, void (*)(b2t_engine*)> e(new b2t_engine(), b2t_engine_destroy);   // destroyed on every error exit
  e->device = dev; e->model = cfg->model; e->pretok = cfg->pretok; e->add_prefix_space = cfg->add_prefix_space;
  cudaDeviceGetAttribute(&e->sm_count, cudaDevAttrMultiProcessorCount, dev);
  if (const char* wc = getenv("B2T_WCACHE")) e->wcache_on = atoi(wc) != 0;
  if (const char* cb = getenv("B2T_CHUNK_BYTES")) {  // host-path chunk size (tests use tiny chunks to exercise the pipeline)
    long long v = atoll(cb);
    if (v >= 1024 && v < (1ll << 31)) e->chunk_bytes = (size_t)v;
  }
  int rc = B2T_OK;
  if ((rc = upload(e->d_cls, ht.cls_packed)) || (rc = upload(e->d_byte_to_id, ht.byte_to_id)) || (rc = upload(e->d_merge, ht.merge_tbl)) ||
      (rc = upload(e->d_word, ht.word_tbl)) || (rc = upload(e->d_pool, ht.word_pool)) || (rc = upload(e->d_edge, ht.edge_tbl)) ||
      (rc = upload(e->d_tok2, ht.tok2_bits)) || (rc = upload(e->d_tri, ht.tri_bits)))
    return rc;
  if (cfg->bert_normalizer & B2T_NORM_BERT) {
    NormHost nh;
    build_bert_norm((cfg->bert_normalizer & B2T_NORM_CLEAN_TEXT) != 0, (cfg->bert_normalizer & B2T_NORM_CHINESE_CHARS) != 0,
                    (cfg->bert_normalizer & B2T_NORM_STRIP_ACCENTS) != 0, (cfg->bert_normalizer & B2T_NORM_LOWERCASE) != 0, &nh);
    if (!nh.ok) return fail(B2T_ERR_UNSUPPORTED, "BertNormalizer table: an image exceeds three bytes per input byte");
    if ((rc = upload(e->d_nt_blk, nh.blk)) || (rc = upload(e->d_nt_ent, nh.ent)) || (rc = upload(e->d_nt_pool, nh.pool)) || (rc = upload(e->d_nt_ascii, nh.ascii)))
      return rc;
    e->nt.blk = e->d_nt_blk.as<uint16_t>(); e->nt.ent = e->d_nt_ent.as<uint32_t>(); e->nt.pool = e->d_nt_pool.as<uint8_t>(); e->nt.ascii = e->d_nt_ascii.as<uint8_t>();
    e->norm_on = 1;
  }
  memset(&e->dt, 0, sizeof(e->dt));
  e->dt.byte_to_id = e->d_byte_to_id.as<uint32_t>();
  e->dt.merge_tbl = e->d_merge.as<uint4>();
  e->dt.merge_mask = ht.merge_tbl.empty() ? 0 : (uint32_t)ht.merge_tbl.size() - 1;
  e->dt.word_tbl = e->d_word.as<uint4>();
  e->dt.word_mask = ht.word_tbl.empty() ? 0 : (uint32_t)ht.word_tbl.size() - 1;
  e->dt.word_pool = e->d_pool.as<uint8_t>();
  e->dt.ignore_merges = cfg->ignore_merges ? 1 : 0;
  e->dt.monotone = ht.monotone ? 1 : 0;
  e->dt.tok2_bits = e->d_tok2.as<uint32_t>(); e->dt.tri_bits = e->d_tri.as<uint32_t>();
  e->monotone = e->dt.monotone;
  e->dt.edge_tbl = e->d_edge.as<uint4>();
  e->dt.edge_mask = ht.edge_tbl.empty() ? 0 : (uint32_t)ht.edge_tbl.size() - 1;
  e->dt.unk_id = ht.unk_id;
  e->dt.max_chars = ht.max_chars;
  // the page kernels use ~23 KB of shared memory per block, 8 blocks per SM: leave the rest of the 228 KB pool to L1
  // (the merge-table probes of the merge rounds are read-only loads and hit there)
  cudaFuncSetAttribute(model_tile_kernel<MODEL_BPE>, cudaFuncAttributePreferredSharedMemoryCarveout, 86);
  cudaFuncSetAttribute(model_tile_kernel<MODEL_WORDPIECE>, cudaFuncAttributePreferredSharedMemoryCarveout, 86);
  cudaError_t se = cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking);
  if (se != cudaSuccess) return fail(B2T_ERR_CUDA, "cudaStreamCreate failed: %s", cudaGetErrorString(se));
  *out = e.release();
  return B2T_OK;
}

extern "C" void b2t_engine_destroy(b2t_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  delete e;
}

// ------------------------------------------------------------------------------------------------ device pipeline
struct ctl_block {  // lives in ws.ctl
  uint32_t max_row;   // dense mode: longest row (template included, after truncation)
  uint32_t err;
  unsigned long long total;
  LongCtl lc;
  uint32_t added_used;   // entries of the added-token list pool handed out
  uint32_t pad;
};

static int ensure_long_pool(Workspace& ws, unsigned long long bytes) {
  if (bytes <= ws.pool_cap) return B2T_OK;
  unsigned long long cap = bytes + bytes / 4 + 4096;
  int rc;
  if ((rc = ws.lp_id.ensure(cap * 4)) || (rc = ws.lp_val.ensure(cap * 8)) || (rc = ws.lp_len.ensure(cap * 4)) || (rc = ws.lp_plen.ensure(cap * 4)) ||
      (rc = ws.lp_aux.ensure(cap * 4)) || (rc = ws.lp_out.ensure(cap * 16)))
    return rc;
  ws.pool_cap = cap;
  return B2T_OK;
}

template <int KIND>
static void launch_pretok(b2t_engine* e, const uint8_t* d_bytes, int64_t n, Workspace& ws, cudaStream_t st, bool added) {
  // every warp owns a contiguous range of whole pages; ~4 waves of resident warps
  const int64_t n_chunks = n / CHUNK + 1;
  const int64_t n_kb = (n_chunks + 31) / 32;
  const int64_t resident = (int64_t)e->sm_count * (KIND == PT_LLAMA3 ? K1_WINDOW_MINBLOCKS : K1_LEAN_MINBLOCKS) * (K1_THREADS / 32);
  int64_t kb = (n_kb + resident * 4 - 1) / (resident * 4);
  kb = std::min<int64_t>(128, std::max<int64_t>(2, (kb + 1) & ~1ll));
  const int64_t n_warps = (n_kb + kb - 1) / kb;
  const int64_t grid = (n_warps + (K1_THREADS / 32) - 1) / (K1_THREADS / 32);
  const AddedBits ab{ws.hard_bits.as<uint32_t>(), ws.inner_bits.as<uint32_t>(), ws.added_bits.as<uint32_t>()};
  if constexpr (KIND == PT_LLAMA3) {
    if (added)
      pretok_stream_kernel<KIND, true><<<(unsigned)grid, K1_THREADS, 0, st>>>(d_bytes, n, ws.doc_bits.as<uint32_t>(), e->d_cls.as<uint32_t>(),
                                                                            ws.start_bits.as<uint32_t>(), ws.page_sum.as<uint64_t>(),
                                                                            (int)n_kb, (int)kb, ab);
    else
      pretok_stream_kernel<KIND><<<(unsigned)grid, K1_THREADS, 0, st>>>(d_bytes, n, ws.doc_bits.as<uint32_t>(), e->d_cls.as<uint32_t>(),
                                                                      ws.start_bits.as<uint32_t>(), ws.page_sum.as<uint64_t>(),
                                                                      (int)n_kb, (int)kb);
  } else {
    const SwapMasks masks{0x55555555u, 0x33333333u, 0x0F0F0F0Fu};
    if (added)
      pretok_lean_kernel<KIND, true><<<(unsigned)grid, K1_THREADS, 0, st>>>(d_bytes, n, ws.doc_bits.as<uint32_t>(), e->d_cls.as<uint32_t>(),
                                                                          ws.start_bits.as<uint32_t>(), ws.drop_bits.as<uint32_t>(),
                                                                          ws.page_sum.as<uint64_t>(), (int)n_kb, (int)kb, masks, ab);
    else
      pretok_lean_kernel<KIND><<<(unsigned)grid, K1_THREADS, 0, st>>>(d_bytes, n, ws.doc_bits.as<uint32_t>(), e->d_cls.as<uint32_t>(),
                                                                    ws.start_bits.as<uint32_t>(), ws.drop_bits.as<uint32_t>(),
                                                                    ws.page_sum.as<uint64_t>(), (int)n_kb, (int)kb, masks);
  }
}

static void rec(b2t_engine* e, cudaStream_t st, const char* name) {
  // records the event that ENDS kernel `name` (event 0 is recorded before the first kernel)
  if (!e->profiling) return;
  if (name == nullptr) { e->n_rec = 0; cudaEventRecord(e->rec_ev[0], st); return; }
  if (e->n_rec >= MAX_KERNEL_RECORDS) return;
  e->rec_name[e->n_rec] = name;
  cudaEventRecord(e->rec_ev[e->n_rec + 1], st);
  e->n_rec++;
}

static uint32_t dense_round(uint32_t len, uint32_t multiple) {
  if (multiple > 0 && len % multiple) len += multiple - len % multiple;
  return len;
}
// b2t_dense_spec -> DenseReq, checked
static int make_dense_req(const b2t_dense_spec* sp, DenseReq* dq) {
  if (!sp) return fail(B2T_ERR_INVALID, "dense spec is null");
  if (sp->struct_size != sizeof(b2t_dense_spec)) return fail(B2T_ERR_INVALID, "b2t_dense_spec: struct_size mismatch (%u != %zu)", sp->struct_size, sizeof(b2t_dense_spec));
  if (sp->n_pre > (uint32_t)DENSE_MAX_SPECIAL || sp->n_post > (uint32_t)DENSE_MAX_SPECIAL)
    return fail(B2T_ERR_UNSUPPORTED, "templates with more than %d special tokens on one side are not supported", DENSE_MAX_SPECIAL);
  if ((sp->n_pre && !sp->pre_ids) || (sp->n_post && !sp->post_ids)) return fail(B2T_ERR_INVALID, "dense spec: null special-token list");
  const uint32_t n_special = sp->n_pre + sp->n_post;
  // tokenizer/mod.rs:1272-1283: the sequence is truncated to max_length - n_added_tokens
  if (sp->max_length && sp->max_length < n_special) return fail(B2T_ERR_INVALID, "max_length %u is smaller than the %u special tokens of the template", sp->max_length, n_special);
  memset(&dq->S, 0, sizeof(dq->S));
  dq->S.keep_max = sp->max_length ? sp->max_length - n_special : DENSE_NO_LIMIT;
  dq->S.pad_id = sp->pad_id; dq->S.n_pre = sp->n_pre; dq->S.n_post = sp->n_post;
  dq->S.trunc_left = sp->truncate_left ? 1 : 0; dq->S.pad_left = sp->pad_left ? 1 : 0;
  for (uint32_t i = 0; i < sp->n_pre; ++i) dq->S.pre[i] = sp->pre_ids[i];
  for (uint32_t i = 0; i < sp->n_post; ++i) dq->S.post[i] = sp->post_ids[i];
  dq->batch_longest = sp->length == 0;
  dq->multiple = sp->pad_to_multiple_of;
  dq->S.L = dq->batch_longest ? 0u : dense_round(sp->length, dq->multiple);
  dq->want_mask = sp->want_mask != 0;
  return B2T_OK;
}

// CSR of the workspace -> dense rows in ws.dense_* (asynchronous on st)
static int launch_dense(b2t_engine* e, Workspace& ws, uint32_t n_docs, const DenseReq& dq, cudaStream_t st) {
  int rc;
  const size_t cells = (size_t)n_docs * dq.S.L;
  if ((rc = ws.dense_ids.ensure(cells * 4 + 16)) || (rc = ws.dense_len.ensure((size_t)n_docs * 4 + 16)) ||
      (dq.want_mask && (rc = ws.dense_mask.ensure(cells + 16))))
    return rc;
  if (n_docs && dq.S.L)
    dense_rows_kernel<<<(unsigned)(((uint64_t)n_docs * 32 + 255) / 256), 256, 0, st>>>(
        ws.ids.as<uint32_t>(), ws.row_ptr.as<uint64_t>(), n_docs, dq.S, ws.dense_ids.as<uint32_t>(),
        dq.want_mask ? ws.dense_mask.as<uint8_t>() : nullptr, ws.dense_len.as<uint32_t>(), nullptr);
  e->last_launches++;
  CU(cudaGetLastError());
  return B2T_OK;
}

// pass 2 of the model pass: provisional slots -> CSR at the given destination, row_ptr = token_base + shard-local row_ptr
static int finish_device(b2t_engine* e, Workspace& ws, uint32_t* d_ids, uint32_t* d_off, uint32_t* d_wid, uint64_t* d_rp,
                         unsigned long long token_base, cudaStream_t st) {
  const uint32_t flags = ws.req.flags, n_docs = ws.batch.n_docs;
  const int64_t n_pages = ws.batch.n / PAGE + 1;
  compact_kernel<<<(unsigned)((n_pages * 32 + 255) / 256), 256, 0, st>>>(
      ws.tile_count.as<uint32_t>(), ws.tile_first.as<uint32_t>(), ws.tile_lexcl.as<unsigned long long>(), ws.tile_bsum.as<unsigned long long>(), n_pages,
      ws.tmp_ids.as<uint32_t>(), (flags & B2T_WANT_OFFSETS) ? ws.tmp_offsets.as<uint2>() : nullptr,
      (flags & B2T_WANT_WORD_IDS) ? ws.tmp_word_ids.as<uint32_t>() : nullptr, d_ids,
      (flags & B2T_WANT_OFFSETS) ? reinterpret_cast<uint2*>(d_off) : nullptr, (flags & B2T_WANT_WORD_IDS) ? d_wid : nullptr);
  row_ptr_fix_kernel<<<(n_docs + 1 + 255) / 256, 256, 0, st>>>(ws.batch.doc_off, n_docs, ws.tile_lexcl.as<unsigned long long>(),
                                                             ws.tile_bsum.as<unsigned long long>(), ws.row_ptr_local.as<uint64_t>(), d_rp, token_base);
  e->last_launches += 2;
  if (ws.norm_active && (flags & B2T_WANT_OFFSETS) && n_docs)
    norm_offsets_kernel<<<(unsigned)(((uint64_t)n_docs * 32 + 255) / 256), 256, 0, st>>>(d_rp, n_docs, token_base, ws.nrm_doc_off.as<uint64_t>(), ws.nrm_doc_char0.as<uint32_t>(),
                                                                                      ws.nrm_src_char.as<uint32_t>(), reinterpret_cast<uint2*>(d_off));
  CU(cudaGetLastError());
  return B2T_OK;
}

// bpe_tile on the 1 GB corpus, H100 80GB HBM3 at a 400 W power limit: 2^19 slots 19.7 ms, 2^20 18.6, 2^21 17.4-17.5,
// 2^22 17.1; 2^21 x 64 B = 128 MiB
constexpr uint32_t WCACHE_SLOTS = 1u << 21;

// ---- the stages of run_device_pipeline, in the order it calls them

// add_prefix_space: re-pack the batch with the prefix spaces inserted (byte_level.rs:121-125); costs one small host sync
// for the new size
static int repack_prefix(b2t_engine* e, Workspace& ws, Batch& b, cudaStream_t st) {
  if (!e->add_prefix_space || b.n_docs == 0 || b.n == 0) return B2T_OK;
  const uint8_t* d_bytes = b.bytes; const uint64_t* d_doc_off = b.doc_off; const int64_t n = b.n; const uint32_t n_docs = b.n_docs;
  int rc;
  const int64_t cap = n + n_docs + 64;
  const uint32_t nb = (n_docs + PFX_BLOCK - 1) / PFX_BLOCK;
  if ((rc = ws.pfx_bytes.ensure(cap)) || (rc = ws.pfx_doc_off.ensure(((size_t)n_docs + 1) * 8)) || (rc = ws.pfx_local.ensure((size_t)n_docs * 4)) ||
      (rc = ws.pfx_block.ensure((size_t)nb * 4 + 16)) || (rc = ws.prefix_bits.ensure((cap / 32 + 2) * 4)) || (rc = ws.pfx_total.ensure(16)) ||
      (rc = ws.h_ctl.ensure(sizeof(ctl_block), false)))
    return rc;
  CU(cudaMemsetAsync(ws.prefix_bits.p, 0, (cap / 32 + 2) * 4, st));
  pfx_scan_block_kernel<<<nb, PFX_BLOCK, 0, st>>>(d_bytes, d_doc_off, n_docs, ws.pfx_local.as<uint32_t>(), ws.pfx_block.as<uint32_t>());
  pfx_scan_top_kernel<<<1, PFX_BLOCK, 0, st>>>(ws.pfx_block.as<uint32_t>(), nb, ws.pfx_total.as<unsigned long long>());
  pfx_offsets_kernel<<<(n_docs + 1 + 255) / 256, 256, 0, st>>>(d_bytes, d_doc_off, n_docs, ws.pfx_local.as<uint32_t>(), ws.pfx_block.as<uint32_t>(),
                                                              ws.pfx_total.as<unsigned long long>(), ws.pfx_doc_off.as<uint64_t>(), ws.prefix_bits.as<uint32_t>());
  pfx_copy_kernel<<<(unsigned)(((int64_t)n_docs * 32 + 255) / 256), 256, 0, st>>>(d_bytes, d_doc_off, ws.pfx_doc_off.as<uint64_t>(), n_docs, ws.pfx_bytes.as<uint8_t>());
  unsigned long long added = 0;
  CU(cudaMemcpyAsync(&added, ws.pfx_total.p, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  b.bytes = ws.pfx_bytes.as<uint8_t>(); b.doc_off = ws.pfx_doc_off.as<uint64_t>(); b.n += (int64_t)added;
  b.prefix_bits = ws.prefix_bits.as<uint32_t>();
  return B2T_OK;
}

// N1-N2 BertNormalizer as a byte-rewriting pre-pass: the kernels after it see the normalized batch, the offsets are mapped
// back at the end (N3 in finish_device); costs one small host sync for the size of the normalized batch
static int normalize(b2t_engine* e, Workspace& ws, Batch& b, uint32_t flags, cudaStream_t st) {
  ws.norm_active = false;
  if (!e->norm_on || b.n == 0 || b.n_docs == 0) return B2T_OK;
  const uint8_t* d_bytes = b.bytes; const uint64_t* d_doc_off = b.doc_off; const int64_t n = b.n; const uint32_t n_docs = b.n_docs;
  int rc;
  if (flags & B2T_OFFSETS_BYTES) return fail(B2T_ERR_UNSUPPORTED, "byte offsets are not available behind a normalizer (character offsets are)");
  const int64_t o_words = n / 32 + 2, o_pages = n / PAGE + 1, o_blk = (o_pages + TSCAN - 1) / TSCAN;
  if ((rc = ws.nrm_doc_bits.ensure(o_words * 4)) || (rc = ws.nrm_pfd.ensure(o_pages * 4)) || (rc = ws.nrm_page_out.ensure(o_pages * 4)) ||
      (rc = ws.nrm_page_chars.ensure(o_pages * 4)) || (rc = ws.nrm_lexcl_o.ensure(o_pages * 8)) || (rc = ws.nrm_lexcl_c.ensure(o_pages * 8)) ||
      (rc = ws.nrm_bsum_o.ensure((o_blk + 2) * 8)) || (rc = ws.nrm_bsum_c.ensure((o_blk + 2) * 8)) || (rc = ws.nrm_tot.ensure(32)) ||
      (rc = ws.nrm_doc_off.ensure(((size_t)n_docs + 1) * 8)) || (rc = ws.nrm_doc_char0.ensure(((size_t)n_docs + 1) * 4)) || (rc = ws.h_ctl.ensure(sizeof(ctl_block), false)))
    return rc;
  CU(cudaMemsetAsync(ws.nrm_doc_bits.p, 0, o_words * 4, st));
  CU(cudaMemsetAsync(ws.nrm_tot.p, 0, 32, st));
  rec(e, st, nullptr);
  unsigned long long* tot = ws.nrm_tot.as<unsigned long long>();
  uint32_t* nerr = reinterpret_cast<uint32_t*>(tot + 2);
  doc_mark_kernel<<<(n_docs + 1 + 255) / 256, 256, 0, st>>>(d_doc_off, n_docs, ws.nrm_doc_bits.as<uint32_t>(), ws.nrm_pfd.as<uint32_t>());
  norm_count_kernel<<<(unsigned)o_pages, NORM_THREADS, 0, st>>>(d_bytes, n, e->nt, ws.nrm_page_out.as<uint32_t>(), ws.nrm_page_chars.as<uint32_t>(), nerr);
  tile_scan_block_kernel<<<(unsigned)o_blk, TSCAN, 0, st>>>(ws.nrm_page_out.as<uint32_t>(), ws.nrm_lexcl_o.as<unsigned long long>(), ws.nrm_bsum_o.as<unsigned long long>(), o_pages);
  tile_scan_top_kernel<<<1, TSCAN, 0, st>>>(ws.nrm_bsum_o.as<unsigned long long>(), o_blk, tot);
  tile_scan_block_kernel<<<(unsigned)o_blk, TSCAN, 0, st>>>(ws.nrm_page_chars.as<uint32_t>(), ws.nrm_lexcl_c.as<unsigned long long>(), ws.nrm_bsum_c.as<unsigned long long>(), o_pages);
  tile_scan_top_kernel<<<1, TSCAN, 0, st>>>(ws.nrm_bsum_c.as<unsigned long long>(), o_blk, tot + 1);
  e->last_launches += 6;
  unsigned long long h_tot[3] = {0, 0, 0};
  CU(cudaMemcpyAsync(h_tot, ws.nrm_tot.p, 24, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));   // one small read: the size of the normalized batch
  if ((uint32_t)h_tot[2] & ERR_NORM_UNSUPPORTED)
    return fail(B2T_ERR_UNSUPPORTED, "the text holds a combining character that strip_accents keeps right behind another combining character: "
                "their canonical order (NFD) is not restated on the device");
  const int64_t m = (int64_t)h_tot[0];
  if (m + (int64_t)n_docs >= (1ll << 31)) return fail(B2T_ERR_TOO_LARGE, "normalized batch of %lld bytes exceeds the per-call limit of 2^31-1; split it", (long long)m);
  if ((rc = ws.nrm_bytes.ensure((size_t)m + 64)) || (rc = ws.nrm_src_char.ensure(((size_t)m + 1) * 4))) return rc;
  norm_write_kernel<<<(unsigned)o_pages, NORM_THREADS, 0, st>>>(d_bytes, n, e->nt, ws.nrm_lexcl_o.as<unsigned long long>(), ws.nrm_bsum_o.as<unsigned long long>(),
                                                             ws.nrm_lexcl_c.as<unsigned long long>(), ws.nrm_bsum_c.as<unsigned long long>(), TSCAN,
                                                             ws.nrm_pfd.as<uint32_t>(), d_doc_off, n_docs, ws.nrm_bytes.as<uint8_t>(), ws.nrm_src_char.as<uint32_t>(),
                                                             ws.nrm_doc_off.as<uint64_t>(), ws.nrm_doc_char0.as<uint32_t>(), nerr);
  e->last_launches++;
  CU(cudaGetLastError());
  rec(e, st, "normalize");
  b.bytes = ws.nrm_bytes.as<uint8_t>(); b.doc_off = ws.nrm_doc_off.as<uint64_t>(); b.n = m;
  ws.norm_active = true;
  return B2T_OK;
}

// Sizes the workspace for the batch the kernels run on and clears what they accumulate into.
static int size_buffers(b2t_engine* e, Workspace& ws, const Batch& b, uint32_t flags, bool model_pass, cudaStream_t st) {
  const int64_t n = b.n; const uint32_t n_docs = b.n_docs;
  int rc;
  const int64_t n_words = n / 32 + 2, n_pages = n / PAGE + 1;
  if ((rc = ws.doc_bits.ensure(n_words * 4)) || (rc = ws.start_bits.ensure(n_words * 4)) || (rc = ws.page_sum.ensure(n_pages * 8)) ||
      (rc = ws.page_carry.ensure(n_pages * 8)) || (rc = ws.block_sum.ensure((n_pages / SCAN_BLOCK + 2) * 8)) ||
      (rc = ws.block_carry.ensure((n_pages / SCAN_BLOCK + 2) * 8)) || (rc = ws.page_first_doc.ensure(n_pages * 4)) ||
      (rc = ws.ctl.ensure(sizeof(ctl_block))) || (rc = ws.h_ctl.ensure(sizeof(ctl_block), false)))
    return rc;
  if (pretok_drops_whitespace(e->pretok) && (rc = ws.drop_bits.ensure(n_words * 4))) return rc;
  const bool bpe = e->model == B2T_MODEL_BPE;
  if (model_pass && (rc = ws.wcache.ensure((size_t)WCACHE_SLOTS * 64))) return rc;
  if (model_pass && bpe) {
    if ((rc = ws.page_long.ensure(n_pages * 4)) || (rc = ws.long_desc.ensure((size_t)(n / (LONG_PRETOK_MIN + 1) + 2) * sizeof(LongDesc))) ||
        (rc = ws.long_desc1.ensure((size_t)(n / (LONG_PRETOK_MIN + 1) + 2) * sizeof(LongDesc))) || (rc = ws.soft_bits.ensure(n_words * 4)) ||
        (rc = ws.page_soft.ensure(n_pages)) || (rc = ensure_long_pool(ws, 1u << 20)))
      return rc;
  }
  if (model_pass) {
    if ((rc = ws.ids.ensure((size_t)(n + 1) * 4)) || (rc = ws.tmp_ids.ensure((size_t)(n + 1) * 4)) || (rc = ws.row_ptr.ensure(((size_t)n_docs + 1) * 8)) || (rc = ws.row_ptr_local.ensure(((size_t)n_docs + 1) * 8)) ||
        (rc = ws.tile_count.ensure(n_pages * 4)) || (rc = ws.tile_first.ensure(n_pages * 4)) || (rc = ws.tile_lexcl.ensure(n_pages * 8)) ||
        (rc = ws.tile_bsum.ensure((n_pages / TSCAN + 2) * 8)))
      return rc;
    if ((flags & B2T_WANT_OFFSETS) && ((rc = ws.offsets.ensure((size_t)(n + 1) * 8)) || (rc = ws.tmp_offsets.ensure((size_t)(n + 1) * 8)))) return rc;
    if ((flags & B2T_WANT_WORD_IDS) && ((rc = ws.word_ids.ensure((size_t)(n + 1) * 4)) || (rc = ws.tmp_word_ids.ensure((size_t)(n + 1) * 4)))) return rc;
  }
  if (e->has_added && !(flags & B2T_NO_ADDED_TOKENS)) {
    if (e->add_prefix_space) return fail(B2T_ERR_UNSUPPORTED, "added-token extraction on the device does not combine with add_prefix_space (the prefix goes in front of every piece)");
    if ((rc = ws.cand0.ensure(n_words * 4)) || (rc = ws.cand1.ensure(n_words * 4)) || (rc = ws.cand_any.ensure((n_words / 32 + 2) * 4)) || (rc = ws.hard_bits.ensure(n_words * 4)) ||
        (rc = ws.inner_bits.ensure(n_words * 4)) || (rc = ws.added_bits.ensure(n_words * 4)) ||
        (rc = ws.added_head.ensure(n_pages * 4)) || (rc = ws.added_pool.ensure((size_t)(n / 16 + 4096) * 8)))
      return rc;
    ws.added_cap = (uint32_t)(n / 16 + 4096);
    CU(cudaMemsetAsync(ws.inner_bits.p, 0, n_words * 4, st));
    CU(cudaMemsetAsync(ws.added_bits.p, 0, n_words * 4, st));
    CU(cudaMemsetAsync(ws.added_head.p, 0xFF, n_pages * 4, st));
  }
  CU(cudaMemsetAsync(ws.doc_bits.p, 0, n_words * 4, st));
  CU(cudaMemsetAsync(ws.ctl.p, 0, sizeof(ctl_block), st));
  if (model_pass) CU(cudaMemsetAsync(ws.wcache.p, 0, (size_t)WCACHE_SLOTS * 64, st));
  if (model_pass && bpe) {
    CU(cudaMemsetAsync(ws.soft_bits.p, 0, n_words * 4, st));
    CU(cudaMemsetAsync(ws.page_soft.p, 0, n_pages, st));
  }
  return B2T_OK;
}

// K0 doc_mark, [A1-A2 added-token extraction,] K1 pretok_scan, K1b page_scan
static int scan(b2t_engine* e, Workspace& ws, const Batch& b, bool added, cudaStream_t st) {
  const uint8_t* d_bytes = b.bytes; const uint64_t* d_doc_off = b.doc_off; const int64_t n = b.n; const uint32_t n_docs = b.n_docs;
  const int64_t n_words = n / 32 + 2, n_pages = n / PAGE + 1, n_chunks_all = n / CHUNK + 1;
  if (!ws.norm_active) rec(e, st, nullptr);
  doc_mark_kernel<<<(n_docs + 1 + 255) / 256, 256, 0, st>>>(d_doc_off, n_docs, ws.doc_bits.as<uint32_t>(), ws.page_first_doc.as<uint32_t>());
  rec(e, st, "doc_mark"); e->last_launches++;
  if (added) {
    // added / special tokens (added_vocabulary.rs:430-564): candidates, then one thread per document that holds one
    ctl_block* ctl = ws.ctl.as<ctl_block>();
    CU(cudaMemcpyAsync(ws.hard_bits.p, ws.doc_bits.p, n_words * 4, cudaMemcpyDeviceToDevice, st));
    added_scan_kernel<<<(unsigned)((n_chunks_all + 255) / 256), 256, 0, st>>>(d_bytes, n, e->at, ws.cand0.as<uint32_t>(), ws.cand1.as<uint32_t>(), ws.cand_any.as<uint32_t>());
    AddedOut ao{ws.hard_bits.as<uint32_t>(), ws.inner_bits.as<uint32_t>(), ws.added_bits.as<uint32_t>(), ws.added_head.as<uint32_t>(),
                ws.added_pool.as<uint2>(), &ctl->added_used, ws.added_cap, &ctl->err};
    added_resolve_kernel<<<(n_docs + 127) / 128, 128, 0, st>>>(d_bytes, d_doc_off, n_docs, e->at, ws.cand0.as<uint32_t>(), ws.cand1.as<uint32_t>(), ws.cand_any.as<uint32_t>(), ao);
    rec(e, st, "added_tokens"); e->last_launches += 2;
  }
  switch (e->pretok) {
    case PT_GPT2: launch_pretok<PT_GPT2>(e, d_bytes, n, ws, st, added); break;
    case PT_LLAMA3: launch_pretok<PT_LLAMA3>(e, d_bytes, n, ws, st, added); break;
    case PT_WHITESPACE: launch_pretok<PT_WHITESPACE>(e, d_bytes, n, ws, st, added); break;
    case PT_BERT: launch_pretok<PT_BERT>(e, d_bytes, n, ws, st, added); break;
    default: launch_pretok<PT_NOREGEX>(e, d_bytes, n, ws, st, added); break;
  }
  rec(e, st, "pretok_scan"); e->last_launches++;
  const int64_t n_scan_blocks = (n_pages + SCAN_BLOCK - 1) / SCAN_BLOCK;
  page_scan_block_kernel<<<(unsigned)n_scan_blocks, SCAN_BLOCK, 0, st>>>(ws.page_sum.as<uint64_t>(), ws.page_carry.as<uint64_t>(),
                                                                      ws.block_sum.as<uint64_t>(), n_pages);
  page_scan_top_kernel<<<1, SCAN_BLOCK, 0, st>>>(ws.block_sum.as<uint64_t>(), ws.block_carry.as<uint64_t>(), n_scan_blocks);
  rec(e, st, "page_scan"); e->last_launches += 2;
  return B2T_OK;
}

// K1c / K2L (BPE): find the long pre-tokens, cut them where no token can span, find the pieces that are still long and
// merge those into the long pool
static void long_pretokens(b2t_engine* e, Workspace& ws, const Batch& b, cudaStream_t st) {
  const uint8_t* d_bytes = b.bytes; const int64_t n = b.n;
  const int64_t n_pages = n / PAGE + 1;
  ctl_block* ctl = ws.ctl.as<ctl_block>();
  LongPool pool;
  pool.id = ws.lp_id.as<uint32_t>(); pool.val = ws.lp_val.as<uint64_t>(); pool.len = ws.lp_len.as<uint32_t>(); pool.plen = ws.lp_plen.as<uint32_t>();
  pool.aux = ws.lp_aux.as<uint32_t>(); pool.out = ws.lp_out.as<uint4>(); pool.cap = ws.pool_cap;
  long_find_kernel<0><<<(unsigned)((n_pages + 7) / 8), 256, 0, st>>>(ws.start_bits.as<uint32_t>(), nullptr, nullptr, n, n_pages, &ctl->lc,
                                                                    ws.long_desc1.as<LongDesc>(), nullptr, 0ull);
  soft_cut_kernel<<<(unsigned)(e->sm_count * 4), 256, 0, st>>>(d_bytes, &ctl->lc, ws.long_desc1.as<LongDesc>(), ws.soft_bits.as<uint32_t>(),
                                                             ws.page_soft.as<uint8_t>(), e->dt);
  long_find_kernel<1><<<(unsigned)((n_pages + 7) / 8), 256, 0, st>>>(ws.start_bits.as<uint32_t>(), ws.soft_bits.as<uint32_t>(), ws.page_soft.as<uint8_t>(),
                                                                    n, n_pages, &ctl->lc, ws.long_desc.as<LongDesc>(), ws.page_long.as<int32_t>(), ws.pool_cap);
  rec(e, st, "long_find"); e->last_launches += 3;
  bpe_long_kernel<<<(unsigned)(e->sm_count * 2), LONG_THREADS, 0, st>>>(d_bytes, &ctl->lc, ws.long_desc.as<LongDesc>(), pool, e->dt, e->monotone);
  rec(e, st, "bpe_long"); e->last_launches++;
}

// K2 model_tile into provisional slots, then pass 2's page token counts -> exclusive scan (the total goes to the control block)
static void model_and_count(b2t_engine* e, Workspace& ws, const Batch& b, uint32_t flags, bool added, cudaStream_t st) {
  const int64_t n_pages = b.n / PAGE + 1;
  ModelParams P;
  P.bytes = b.bytes; P.n = b.n;
  P.start_bits = ws.start_bits.as<uint32_t>(); P.drop_bits = ws.drop_bits.as<uint32_t>(); P.doc_bits = ws.doc_bits.as<uint32_t>();
  P.soft_bits = ws.soft_bits.as<uint32_t>(); P.page_soft = ws.page_soft.as<uint8_t>();
  P.page_carry = ws.page_carry.as<uint64_t>(); P.block_carry = ws.block_carry.as<uint64_t>(); P.page_first_doc = ws.page_first_doc.as<uint32_t>();
  P.doc_off = b.doc_off; P.n_docs = b.n_docs;
  P.flags = ((flags & B2T_WANT_OFFSETS) ? F_OFFSETS : 0u) | ((flags & B2T_WANT_WORD_IDS) ? F_WORD_IDS : 0u) |
            (((flags & B2T_OFFSETS_BYTES) || ws.norm_active) ? F_BYTE_OFFSETS : 0u);   // behind the normalizer: bytes of the normalized document, mapped back by norm_offsets_kernel
  P.ids = ws.tmp_ids.as<uint32_t>(); P.offsets = ws.tmp_offsets.as<uint32_t>(); P.word_ids = ws.tmp_word_ids.as<uint32_t>();
  P.row_ptr = ws.row_ptr_local.as<uint64_t>();
  P.tile_count = ws.tile_count.as<uint32_t>(); P.tile_first = ws.tile_first.as<uint32_t>();
  ctl_block* ctl = ws.ctl.as<ctl_block>();
  P.err_flag = &ctl->err;
  P.n_tiles = n_pages;
  P.page_long = ws.page_long.as<int32_t>(); P.long_desc = ws.long_desc.as<LongDesc>(); P.long_out = ws.lp_out.as<uint4>();
  P.wcache = ws.wcache.as<uint4>(); P.wcache_mask = WCACHE_SLOTS - 1; P.wcache_on = e->wcache_on;
  P.prefix_bits = b.prefix_bits;
  P.added_bits = added ? ws.added_bits.as<uint32_t>() : nullptr; P.added_head = ws.added_head.as<uint32_t>(); P.added_pool = ws.added_pool.as<uint2>();
  P.flag_added = (flags & B2T_FLAG_ADDED_IDS) ? 1u : 0u;
  P.t = e->dt;
  if (e->model == B2T_MODEL_BPE) model_tile_kernel<MODEL_BPE><<<(unsigned)n_pages, MODEL_THREADS, 0, st>>>(P);
  else model_tile_kernel<MODEL_WORDPIECE><<<(unsigned)n_pages, MODEL_THREADS, 0, st>>>(P);
  rec(e, st, e->model == B2T_MODEL_BPE ? "bpe_tile" : "wordpiece_tile"); e->last_launches++;
  const int64_t n_tblk = (n_pages + TSCAN - 1) / TSCAN;
  tile_scan_block_kernel<<<(unsigned)n_tblk, TSCAN, 0, st>>>(ws.tile_count.as<uint32_t>(), ws.tile_lexcl.as<unsigned long long>(),
                                                           ws.tile_bsum.as<unsigned long long>(), n_pages);
  tile_scan_top_kernel<<<1, TSCAN, 0, st>>>(ws.tile_bsum.as<unsigned long long>(), n_tblk, &ctl->total);
  e->last_launches += 2;
}

// The compaction into the workspace's CSR (unless the caller finishes into its own buffers), then in dense mode the longest
// row always (the host checks it against L / derives L from it) and the rows themselves now if L is fixed; the control
// block is queued for the host last
static int finish_tail(b2t_engine* e, Workspace& ws, cudaStream_t st) {
  const DenseReq* dq = ws.req.dq;
  const bool finish = ws.req.until == RUN_RESULT;
  const uint32_t n_docs = ws.batch.n_docs;
  int rc;
  if (finish && (rc = finish_device(e, ws, ws.ids.as<uint32_t>(), ws.offsets.as<uint32_t>(), ws.word_ids.as<uint32_t>(), ws.row_ptr.as<uint64_t>(), 0ull, st)))
    return rc;
  rec(e, st, "scan_compact");
  if (dq && finish) {
    ctl_block* ctl = ws.ctl.as<ctl_block>();
    if (n_docs) row_len_max_kernel<<<(n_docs + 255) / 256, 256, 0, st>>>(ws.row_ptr.as<uint64_t>(), n_docs, dq->S.keep_max, dq->S.n_pre + dq->S.n_post, &ctl->max_row);
    e->last_launches++;
    if (!dq->batch_longest && (rc = launch_dense(e, ws, n_docs, *dq, st))) return rc;
    rec(e, st, "dense_rows");
  }
  CU(cudaMemcpyAsync(ws.h_ctl.p, ws.ctl.p, sizeof(ctl_block), cudaMemcpyDeviceToHost, st));
  return B2T_OK;
}

// Runs ws.req, a batch resident on the device, as far as ws.req.until.  Does not synchronise (except for the small host
// reads of the prefix re-pack and the normalizer).  The launch count leaves out the prefix re-pack and N3.
static int run_device_pipeline(b2t_engine* e, Workspace& ws, cudaStream_t st) {
  const Request& q = ws.req;
  if (q.n + (int64_t)q.n_docs >= (1ll << 31)) return fail(B2T_ERR_TOO_LARGE, "batch of %lld bytes exceeds the per-call limit of 2^31-1; split it", (long long)q.n);
  Batch& b = ws.batch;
  b = Batch{q.bytes, q.n, q.doc_off, q.n_docs, nullptr};
  e->last_launches = 0;
  const bool model_pass = q.until != RUN_PRETOK;
  int rc;
  if ((rc = repack_prefix(e, ws, b, st)) || (rc = normalize(e, ws, b, q.flags, st)) || (rc = size_buffers(e, ws, b, q.flags, model_pass, st)))
    return rc;
  const bool added = e->has_added && !(q.flags & B2T_NO_ADDED_TOKENS) && b.n > 0 && b.n_docs > 0;
  if ((rc = scan(e, ws, b, added, st))) return rc;
  if (model_pass) {
    if (e->model == B2T_MODEL_BPE) long_pretokens(e, ws, b, st);
    model_and_count(e, ws, b, q.flags, added, st);
    if ((rc = finish_tail(e, ws, st))) return rc;
  }
  CU(cudaGetLastError());
  return B2T_OK;
}

// Checks the control block of a run the host has waited for.  While the long pool was too small (rare: the batch holds
// more bytes of long pre-tokens than the pool), grows it to what the run asked for and repeats ws.req on st, three runs
// in all.  *reran tells whether the run was repeated.
static int check_run(b2t_engine* e, Workspace& ws, cudaStream_t st, bool* reran = nullptr) {
  for (int attempt = 0;; ++attempt) {
    const ctl_block* c = ws.h_ctl.as<ctl_block>();
    if (c->err & ERR_ADDED_UNSUPPORTED)   // (first: a refused span leaves the later kernels with half of the picture)
      return fail(B2T_ERR_UNSUPPORTED, "added-token extraction: a span over %d bytes, more spans than one per 16 input bytes, or overlapping spans; "
                  "pass B2T_NO_ADDED_TOKENS and split on the host", ADDED_MAX_SPAN);
    if ((c->err | c->lc.err) & ERR_INTERNAL) return fail(B2T_ERR_CUDA, "internal error: long pre-token / added-token bookkeeping mismatch");
    if (!(c->lc.err & ERR_POOL_OVERFLOW)) return B2T_OK;
    if (attempt >= 2) return fail(B2T_ERR_CUDA, "long pool did not converge");
    if (reran) *reran = true;
    int rc;
    if ((rc = ensure_long_pool(ws, c->lc.pool_used)) || (rc = run_device_pipeline(e, ws, st))) return rc;
    CU(cudaStreamSynchronize(st));
  }
}

static int ensure_events(b2t_engine* e) {
  if (e->rec_ev_made) return B2T_OK;
  for (auto& ev : e->rec_ev) CU(cudaEventCreate(&ev));
  e->rec_ev_made = true;
  return B2T_OK;
}

extern "C" int b2t_engine_set_profiling(b2t_engine* e, int on) {
  if (!e) return fail(B2T_ERR_INVALID, "null engine");
  std::lock_guard<std::mutex> lk(e->dev_mu);
  CU(cudaSetDevice(e->device));
  if (on) { int rc = ensure_events(e); if (rc) return rc; }
  e->profiling = on ? 1 : 0;
  e->n_rec = 0;
  return B2T_OK;
}

extern "C" int b2t_engine_last_kernels(const b2t_engine* e, const char** names, float* ms, int cap) {
  if (!e) return 0;
  if (e->profiling && e->n_rec > 0) {
    cudaEventSynchronize(e->rec_ev[e->n_rec]);
    for (int i = 0; i < e->n_rec && i < cap; ++i) {
      if (names) names[i] = e->rec_name[i];
      if (ms) { ms[i] = 0.f; cudaEventElapsedTime(&ms[i], e->rec_ev[i], e->rec_ev[i + 1]); }
    }
  }
  return e->last_launches;
}

// The device-resident entry points: argument checks (and in dense mode the spec, read into *dq), then the whole call under
// dev_mu on the engine's one device workspace, on the caller's stream or the engine's own.  `done(ws, st)` takes the
// finished run after the host has waited for it.
template <class Done>
static int device_encode(const char* fn, b2t_engine* e, const void* out, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off,
                         uint32_t n_docs, uint32_t flags, RunUntil until, const b2t_dense_spec* spec, DenseReq* dq, void* stream, Done&& done) {
  if (!e || !out || !d_doc_off || (!d_bytes && n_bytes)) return fail(B2T_ERR_INVALID, "%s: null argument", fn);
  if (((uintptr_t)d_bytes & 15u) != 0) return fail(B2T_ERR_INVALID, "%s: d_bytes must be 16-byte aligned", fn);
  int rc;
  if (dq && (rc = make_dense_req(spec, dq))) return rc;
  std::lock_guard<std::mutex> lk(e->dev_mu);
  CU(cudaSetDevice(e->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : e->own_stream;
  Workspace& ws = e->dev_ws;
  if (until == RUN_COUNT) ws.pending = false;   // (a failed begin leaves nothing to finish)
  ws.req = Request{d_bytes, (int64_t)n_bytes, d_doc_off, n_docs, flags, until, dq};
  if ((rc = run_device_pipeline(e, ws, st))) return rc;
  CU(cudaStreamSynchronize(st));
  if ((rc = check_run(e, ws, st))) return rc;
  return done(ws, st);
}

extern "C" int b2t_encode_batch_device(b2t_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off,
                                       uint32_t n_docs, uint32_t flags, void* stream, b2t_result** out) {
  return device_encode("b2t_encode_batch_device", e, out, d_bytes, n_bytes, d_doc_off, n_docs, flags, RUN_RESULT, nullptr, nullptr, stream,
                       [&](Workspace& ws, cudaStream_t) -> int {
    b2t_result* r = new b2t_result();
    r->eng = e; r->on_device = 1; r->n_docs = n_docs;
    r->n_tokens = ws.h_ctl.as<ctl_block>()->total;
    r->ids = ws.ids.as<uint32_t>();
    r->offsets = (flags & B2T_WANT_OFFSETS) ? ws.offsets.as<uint32_t>() : nullptr;
    r->word_ids = (flags & B2T_WANT_WORD_IDS) ? ws.word_ids.as<uint32_t>() : nullptr;
    r->row_ptr = ws.row_ptr.as<uint64_t>();
    *out = r;
    return B2T_OK;
  });
}

extern "C" int b2t_encode_batch_device_begin(b2t_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off,
                                             uint32_t n_docs, uint32_t flags, void* stream, uint64_t* n_tokens) {
  return device_encode("b2t_encode_batch_device_begin", e, n_tokens, d_bytes, n_bytes, d_doc_off, n_docs, flags, RUN_COUNT, nullptr, nullptr, stream,
                       [&](Workspace& ws, cudaStream_t) -> int {
    *n_tokens = ws.h_ctl.as<ctl_block>()->total;
    ws.pending = true;
    return B2T_OK;
  });
}

extern "C" int b2t_encode_batch_device_finish(b2t_engine* e, uint32_t* d_ids, uint32_t* d_offsets, uint32_t* d_word_ids,
                                              uint64_t* d_row_ptr, uint64_t token_base, void* stream) {
  if (!e || !d_ids || !d_row_ptr) return fail(B2T_ERR_INVALID, "b2t_encode_batch_device_finish: null argument");
  std::lock_guard<std::mutex> lk(e->dev_mu);
  Workspace& ws = e->dev_ws;
  if (!ws.pending) return fail(B2T_ERR_INVALID, "b2t_encode_batch_device_finish without a matching begin");
  if ((ws.req.flags & B2T_WANT_OFFSETS) && !d_offsets) return fail(B2T_ERR_INVALID, "offsets were requested at begin: d_offsets is null");
  if ((ws.req.flags & B2T_WANT_WORD_IDS) && !d_word_ids) return fail(B2T_ERR_INVALID, "word ids were requested at begin: d_word_ids is null");
  CU(cudaSetDevice(e->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : e->own_stream;
  ws.pending = false;
  return finish_device(e, ws, d_ids, d_offsets, d_word_ids, d_row_ptr, token_base, st);
}

// ------------------------------------------------------------------------------------------------ added vocabulary
extern "C" int b2t_engine_set_added_tokens(b2t_engine* e, uint32_t n_tokens, const uint8_t* bytes, const uint32_t* off, const uint32_t* ids,
                                           const uint8_t* flags) {
  if (!e) return fail(B2T_ERR_INVALID, "null engine");
  std::lock_guard<std::mutex> lk(e->dev_mu);
  CU(cudaSetDevice(e->device));
  e->has_added = 0;
  if (n_tokens == 0) return B2T_OK;
  if (!bytes || !off || !ids || !flags) return fail(B2T_ERR_INVALID, "b2t_engine_set_added_tokens: null argument");
  if (e->add_prefix_space) return fail(B2T_ERR_UNSUPPORTED, "added-token extraction on the device does not combine with add_prefix_space");
  if (e->norm_on) return fail(B2T_ERR_UNSUPPORTED, "added-token extraction on the device runs on the text the engine is given: with a normalizer the host splits first");
  // two sets (normalized == false first), longest token first inside a set (find_matches: leftmost-longest)
  std::vector<uint32_t> order[2];
  for (uint32_t i = 0; i < n_tokens; ++i) {
    const uint32_t len = off[i + 1] - off[i];
    if (len == 0) continue;                                  // added_vocabulary.rs:288-291: empty tokens are ignored
    if (ids[i] >= (1u << 20)) return fail(B2T_ERR_UNSUPPORTED, "added token id %u: ids of 2^20 and above are not supported", ids[i]);
    order[(flags[i] & B2T_ADDED_NORMALIZED) ? 1 : 0].push_back(i);
  }
  std::vector<uint8_t> tb, tf;
  std::vector<uint32_t> to{0u}, ti, first(16, 0u), pair(2 * 2048, 0u);
  uint32_t begin[3] = {0, 0, 0};
  for (int s2 = 0; s2 < 2; ++s2) {
    std::stable_sort(order[s2].begin(), order[s2].end(), [&](uint32_t a, uint32_t b) { return off[a + 1] - off[a] > off[b + 1] - off[b]; });
    begin[s2] = (uint32_t)ti.size();
    for (uint32_t i : order[s2]) {
      const uint8_t* p = bytes + off[i];
      const uint32_t len = off[i + 1] - off[i];
      tb.insert(tb.end(), p, p + len);
      to.push_back((uint32_t)tb.size()); ti.push_back(ids[i]);
      tf.push_back((uint8_t)(((flags[i] & B2T_ADDED_SINGLE_WORD) ? ADDED_SINGLE_WORD : 0) | ((flags[i] & B2T_ADDED_LSTRIP) ? ADDED_LSTRIP : 0) |
                             ((flags[i] & B2T_ADDED_RSTRIP) ? ADDED_RSTRIP : 0)));
      first[8 * s2 + (p[0] >> 5)] |= 1u << (p[0] & 31);
      for (uint32_t b1 = 0; b1 < 256; ++b1) {
        if (len > 1 && b1 != p[1]) continue;
        const uint32_t two = p[0] | (b1 << 8);
        pair[2048 * s2 + (two >> 5)] |= 1u << (two & 31);
      }
    }
  }
  begin[2] = (uint32_t)ti.size();
  if (ti.empty()) return B2T_OK;
  std::vector<uint8_t> cls(0x110000);
  unicode_class_table(1, cls.data());
  std::vector<uint32_t> packed(0x110000 / 16, 0u);
  for (uint32_t c = 0; c < 0x110000; ++c) packed[c >> 4] |= (uint32_t)cls[c] << ((c & 15) * 2);
  int rc;
  if ((rc = upload(e->d_at_bytes, tb)) || (rc = upload(e->d_at_off, to)) || (rc = upload(e->d_at_id, ti)) || (rc = upload(e->d_at_flags, tf)) ||
      (rc = upload(e->d_at_first, first)) || (rc = upload(e->d_at_pair, pair)) || (rc = upload(e->d_cls_rust, packed)))
    return rc;
  e->at.tok_bytes = e->d_at_bytes.as<uint8_t>(); e->at.tok_off = e->d_at_off.as<uint32_t>(); e->at.tok_id = e->d_at_id.as<uint32_t>();
  e->at.tok_flags = e->d_at_flags.as<uint8_t>();
  e->at.set_begin[0] = begin[0]; e->at.set_begin[1] = begin[1]; e->at.set_begin[2] = begin[2];
  e->at.first_bits = e->d_at_first.as<uint32_t>(); e->at.pair_bits = e->d_at_pair.as<uint32_t>(); e->at.cls_rust = e->d_cls_rust.as<uint32_t>();
  e->at.n_first = 0;
  {
    std::vector<uint32_t> fb;
    for (uint32_t b = 0; b < 256; ++b) if (((first[b >> 5] | first[8 + (b >> 5)]) >> (b & 31)) & 1u) fb.push_back(b);
    if (fb.size() <= 4) { e->at.n_first = (uint32_t)fb.size(); for (size_t i = 0; i < fb.size(); ++i) e->at.first_bcast[i] = fb[i] * 0x01010101u; }
  }
  e->has_added = 1;
  return B2T_OK;
}

// ------------------------------------------------------------------------------------------------ dense mode
extern "C" int b2t_encode_batch_dense(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, const b2t_dense_spec* spec,
                                      b2t_result** out);

extern "C" int b2t_encode_batch_dense_device(b2t_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off, uint32_t n_docs,
                                             const b2t_dense_spec* spec, void* stream, b2t_result** out) {
  DenseReq dq;
  return device_encode("b2t_encode_batch_dense_device", e, out, d_bytes, n_bytes, d_doc_off, n_docs, 0u, RUN_RESULT, spec, &dq, stream,
                       [&](Workspace& ws, cudaStream_t st) -> int {
    int rc2;
    const uint32_t max_row = ws.h_ctl.as<ctl_block>()->max_row;
    if (dq.batch_longest) {
      dq.S.L = dense_round(max_row, dq.multiple);
      if ((rc2 = launch_dense(e, ws, n_docs, dq, st))) return rc2;   // asynchronous on st, like the CSR entry point's result
    } else if (max_row > dq.S.L) {
      return fail(B2T_ERR_INVALID, "a row of %u tokens does not fit the dense length %u: enable truncation (the reference returns a longer row here)", max_row, dq.S.L);
    }
    b2t_result* r = new b2t_result();
    r->eng = e; r->on_device = 1; r->n_docs = n_docs;
    r->n_tokens = ws.h_ctl.as<ctl_block>()->total;
    r->dense_len = dq.S.L;
    r->dense_ids = ws.dense_ids.as<uint32_t>(); r->row_len = ws.dense_len.as<uint32_t>();
    r->dense_mask = dq.want_mask ? ws.dense_mask.as<uint8_t>() : nullptr;
    *out = r;
    return B2T_OK;
  });
}

// ------------------------------------------------------------------------------------------------ host pipeline
static b2t_result* pool_get(b2t_engine* e) {
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->pool.empty()) { b2t_result* r = e->pool.back().release(); e->pool.pop_back(); return r; }
  return new b2t_result();
}

static void pool_put(b2t_engine* e, b2t_result* r) {
  std::lock_guard<std::mutex> lk(e->mu);
  e->pool.emplace_back(r);
}

// A slot set for one host-path call; blocks while MAX_SLOT_SETS calls are in flight.
struct SetLease {
  b2t_engine* e; b2t_engine::SlotSet* ss;
  explicit SetLease(b2t_engine* e_) : e(e_), ss(nullptr) {
    std::unique_lock<std::mutex> lk(e->mu);
    while (true) {
      for (auto& c : e->sets) if (!c->busy) { ss = c.get(); break; }
      if (ss) break;
      if (e->sets.size() < MAX_SLOT_SETS) { e->sets.emplace_back(new b2t_engine::SlotSet()); ss = e->sets.back().get(); break; }
      e->set_free.wait(lk);
    }
    ss->busy = true;
  }
  ~SetLease() {
    { std::lock_guard<std::mutex> lk(e->mu); ss->busy = false; }
    e->set_free.notify_one();
  }
};

static int slot_init(Workspace& ws) {
  if (!ws.stream) CU(cudaStreamCreateWithFlags(&ws.stream, cudaStreamNonBlocking));
  if (!ws.done) CU(cudaEventCreateWithFlags(&ws.done, cudaEventDisableTiming));
  return B2T_OK;
}

// rebases doc offsets of a chunk to the chunk start (runs on the slot's stream before K0)
__global__ void rebase_kernel(uint64_t* doc_off, uint32_t count, uint64_t base) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) doc_off[i] -= base;
}

struct Chunk { uint32_t d0, d1; uint64_t b0, b1; uint64_t tok_base; };

// Queues the copy of a chunk's dense rows (documents d0 .. d0 + nd - 1) into the pinned result, on the slot's stream.
static int queue_dense_copy(b2t_result* r, const Workspace& ws, uint32_t d0, uint32_t nd, const DenseReq& dq) {
  const size_t L = dq.S.L;
  if (nd && L) {
    CU(cudaMemcpyAsync(r->h_dense_ids.as<uint32_t>() + (size_t)d0 * L, ws.dense_ids.p, (size_t)nd * L * 4, cudaMemcpyDeviceToHost, ws.stream));
    if (dq.want_mask) CU(cudaMemcpyAsync(r->h_dense_mask.as<uint8_t>() + (size_t)d0 * L, ws.dense_mask.p, (size_t)nd * L, cudaMemcpyDeviceToHost, ws.stream));
  }
  if (nd) CU(cudaMemcpyAsync(r->h_row_len.as<uint32_t>() + d0, ws.dense_len.p, (size_t)nd * 4, cudaMemcpyDeviceToHost, ws.stream));
  return B2T_OK;
}

static int host_encode(b2t_engine* e, b2t_engine::SlotSet& ss, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, uint32_t flags,
                       b2t_result** out, const DenseReq* dq_in = nullptr) {
  const uint64_t total_bytes = doc_off[n_docs];
  // ---- split into chunks of whole documents
  std::vector<Chunk> chunks;
  uint64_t max_chunk = 0;
  DenseReq dq_local;
  DenseReq* dq = nullptr;
  if (dq_in) { dq_local = *dq_in; dq = &dq_local; flags = 0; }
  // BatchLongest padding needs every row length before the first row can be written: the batch runs as one chunk
  if (dq && dq->batch_longest && total_bytes + n_docs >= (1ull << 31))
    return fail(B2T_ERR_UNSUPPORTED, "dense output padded to the longest row needs the batch in one device pass (< 2^31 bytes); pad to a fixed length instead");
  const uint64_t chunk_bytes = (dq && dq->batch_longest) ? (1ull << 31) : (uint64_t)e->chunk_bytes;
  {
    uint32_t d = 0;
    while (d < n_docs) {
      uint64_t limit = doc_off[d] + chunk_bytes;
      uint32_t d1 = (uint32_t)(std::upper_bound(doc_off + d + 1, doc_off + n_docs + 1, limit) - doc_off) - 1;
      if (d1 <= d) d1 = d + 1;  // a single document larger than the chunk size
      if (doc_off[d1] - doc_off[d] >= (1ull << 31)) return fail(B2T_ERR_TOO_LARGE, "document %u is larger than 2 GiB", d);
      chunks.push_back({d, d1, doc_off[d], doc_off[d1], 0});
      max_chunk = std::max(max_chunk, doc_off[d1] - doc_off[d]);
      d = d1;
    }
    if (chunks.empty()) chunks.push_back({0, 0, 0, 0, 0});
  }
  b2t_result* r = pool_get(e);
  r->eng = e; r->on_device = 0; r->n_docs = n_docs; r->n_tokens = 0;
  int rc;
  const bool want_off = (flags & B2T_WANT_OFFSETS) != 0, want_wid = (flags & B2T_WANT_WORD_IDS) != 0;
  // initial capacity guess: 0.30 tokens per byte, grown on demand (pinned pool => steady state allocates nothing)
  uint64_t cap_tok = std::max<uint64_t>(total_bytes * 3 / 10 + 1024, 4096);
  if ((rc = r->h_row_ptr.ensure(((size_t)n_docs + 1) * 8, false))) { pool_put(e, r); return rc; }
  auto grow = [&](uint64_t need_tok) -> int {
    int rc2;
    if ((rc2 = r->h_ids.ensure(need_tok * 4, true))) return rc2;
    if (want_off && (rc2 = r->h_offsets.ensure(need_tok * 8, true))) return rc2;
    if (want_wid && (rc2 = r->h_word_ids.ensure(need_tok * 4, true))) return rc2;
    return B2T_OK;
  };
  r->dense_len = 0; r->dense_ids = nullptr; r->dense_mask = nullptr; r->row_len = nullptr;
  auto dense_host = [&](uint32_t L) -> int {   // pinned rows of the whole batch
    int rc2;
    const size_t cells = (size_t)n_docs * L;
    if ((rc2 = r->h_dense_ids.ensure(cells * 4 + 16, false)) || (rc2 = r->h_row_len.ensure((size_t)n_docs * 4 + 16, false)) ||
        (dq->want_mask && (rc2 = r->h_dense_mask.ensure(cells + 16, false))))
      return rc2;
    return B2T_OK;
  };
  if (dq) { if (!dq->batch_longest && (rc = dense_host(dq->S.L))) { pool_put(e, r); return rc; } }
  else if ((rc = grow(cap_tok))) { pool_put(e, r); return rc; }

  uint64_t tok_base = 0;
  const size_t nc = chunks.size();
  size_t drained = 0;
  // Pipeline over NSLOT device slots: chunk i is issued (H2D + kernels + count read-back) while older chunks compute;
  // drain(i) waits for chunk i's kernels and queues the D2H of its results on the same slot stream.
  auto drain = [&](size_t ci) -> int {
    Chunk& c = chunks[ci];
    Workspace& ws = ss.slot[ci % NSLOT];
    CU(cudaEventSynchronize(ws.done));
    int rc2;
    bool reran = false;   // (a rerun finds the chunk's input still resident in the slot)
    if ((rc2 = check_run(e, ws, ws.stream, &reran))) return rc2;
    const uint64_t nt = ws.h_ctl.as<ctl_block>()->total;
    c.tok_base = tok_base;
    if (dq) {
      const uint32_t nd = c.d1 - c.d0, max_row = ws.h_ctl.as<ctl_block>()->max_row;
      if (dq->batch_longest) {   // one chunk: L is known now
        dq->S.L = dense_round(max_row, dq->multiple);
        if ((rc2 = dense_host(dq->S.L)) || (rc2 = launch_dense(e, ws, nd, *dq, ws.stream))) return rc2;
      } else if (max_row > dq->S.L) {
        return fail(B2T_ERR_INVALID, "a row of %u tokens does not fit the dense length %u: enable truncation (the reference returns a longer row here)", max_row, dq->S.L);
      }
      // (a fixed length: the rows were queued for the copy right behind the kernels, see issue(); a rerun has replaced them)
      if ((dq->batch_longest || reran) && (rc2 = queue_dense_copy(r, ws, c.d0, nd, *dq))) return rc2;
      tok_base += nt;
      return B2T_OK;
    }
    if (tok_base + nt > cap_tok) {
      // earlier chunks may still be copying into the old buffers: let them land, then grow (contents are kept)
      for (auto& s : ss.slot) if (s.stream) CU(cudaStreamSynchronize(s.stream));
      cap_tok = (tok_base + nt) * 2;
      if ((rc2 = grow(cap_tok))) return rc2;
    }
    const uint32_t nd = c.d1 - c.d0;
    if (nt) {
      CU(cudaMemcpyAsync(r->h_ids.as<uint32_t>() + tok_base, ws.ids.p, nt * 4, cudaMemcpyDeviceToHost, ws.stream));
      if (want_off) CU(cudaMemcpyAsync(r->h_offsets.as<uint32_t>() + 2 * tok_base, ws.offsets.p, nt * 8, cudaMemcpyDeviceToHost, ws.stream));
      if (want_wid) CU(cudaMemcpyAsync(r->h_word_ids.as<uint32_t>() + tok_base, ws.word_ids.p, nt * 4, cudaMemcpyDeviceToHost, ws.stream));
    }
    // chunk-relative row_ptr: entries d0..d1-1 (the last chunk also owns entry d1 = n_docs)
    const size_t nrp = (size_t)nd + (ci + 1 == nc ? 1 : 0);
    if (nrp) CU(cudaMemcpyAsync(r->h_row_ptr.as<uint64_t>() + c.d0, ws.row_ptr.p, nrp * 8, cudaMemcpyDeviceToHost, ws.stream));
    tok_base += nt;
    return B2T_OK;
  };
  auto issue = [&](size_t ci) -> int {
    Workspace& ws = ss.slot[ci % NSLOT];
    int rc2;
    if ((rc2 = slot_init(ws))) return rc2;
    if (ci >= NSLOT) {
      // slot reuse: the chunk that used it must be drained and its copies must have landed
      while (drained + NSLOT <= ci) if ((rc2 = drain(drained++))) return rc2;
      CU(cudaStreamSynchronize(ws.stream));
    }
    const Chunk& c = chunks[ci];
    const uint64_t nb = c.b1 - c.b0;
    const uint32_t nd = c.d1 - c.d0;
    if ((rc2 = ws.bytes.ensure(nb + 64)) || (rc2 = ws.doc_off.ensure(((size_t)nd + 1) * 8))) return rc2;
    if (nb) CU(cudaMemcpyAsync(ws.bytes.p, bytes + c.b0, nb, cudaMemcpyHostToDevice, ws.stream));
    CU(cudaMemcpyAsync(ws.doc_off.p, doc_off + c.d0, ((size_t)nd + 1) * 8, cudaMemcpyHostToDevice, ws.stream));
    if (c.b0) rebase_kernel<<<(nd + 1 + 255) / 256, 256, 0, ws.stream>>>(ws.doc_off.as<uint64_t>(), nd + 1, c.b0);
    ws.req = Request{ws.bytes.as<uint8_t>(), (int64_t)nb, ws.doc_off.as<uint64_t>(), nd, flags, RUN_RESULT, dq};
    if ((rc2 = run_device_pipeline(e, ws, ws.stream))) return rc2;
    // dense rows of a fixed length: their place in the result does not depend on anything the host has to read first, so
    // the copy back is queued right behind the kernels (the CSR modes need the chunk's token count for that)
    if (dq && !dq->batch_longest && (rc2 = queue_dense_copy(r, ws, c.d0, nd, *dq))) return rc2;
    CU(cudaEventRecord(ws.done, ws.stream));
    return B2T_OK;
  };
  // (a failure in either step must reach the common cleanup below: the pooled result goes back, slot streams are drained)
  rc = B2T_OK;
  for (size_t ci = 0; ci < nc && rc == B2T_OK; ++ci) {
    rc = issue(ci);
    // keep at most NSLOT - 1 chunks un-drained so that result copies overlap the next chunks' kernels
    while (rc == B2T_OK && drained + (NSLOT - 1) <= ci) rc = drain(drained++);
  }
  while (rc == B2T_OK && drained < nc) rc = drain(drained++);
  for (auto& s : ss.slot) if (s.stream) cudaStreamSynchronize(s.stream);
  if (rc) { pool_put(e, r); return rc; }

  if (dq) {
    if (n_docs == 0 && dq->batch_longest) dq->S.L = 0;
    r->n_tokens = tok_base; r->ids = nullptr; r->offsets = nullptr; r->word_ids = nullptr; r->row_ptr = nullptr;
    r->dense_len = dq->S.L;
    r->dense_ids = r->h_dense_ids.as<uint32_t>(); r->row_len = r->h_row_len.as<uint32_t>();
    r->dense_mask = dq->want_mask ? r->h_dense_mask.as<uint8_t>() : nullptr;
  } else {
    // chunk-relative row_ptr -> batch-relative (host fix-up: one addition per document)
    uint64_t* rp = r->h_row_ptr.as<uint64_t>();
    for (size_t ci = 1; ci < nc; ++ci) {
      const Chunk& c = chunks[ci];
      const uint32_t hi = (ci + 1 == nc) ? c.d1 : c.d1 - 1;
      for (uint32_t d = c.d0; d <= hi; ++d) rp[d] += c.tok_base;
    }
    r->n_tokens = tok_base;
    r->ids = r->h_ids.as<uint32_t>();
    r->offsets = want_off ? r->h_offsets.as<uint32_t>() : nullptr;
    r->word_ids = want_wid ? r->h_word_ids.as<uint32_t>() : nullptr;
    r->row_ptr = rp;
  }
  *out = r;
  return B2T_OK;
}

// The host-buffer entry points: argument checks (and in dense mode the spec, read into *dq), then `run(slot set)` on a slot
// set of the call's own -- and, while per-kernel profiling is on, on the whole engine (the event records are one per engine).
template <class Run>
static int host_call(const char* fn, b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, b2t_result** out,
                     const b2t_dense_spec* spec, DenseReq* dq, Run&& run) {
  if (!e || !out || !doc_off || (!bytes && doc_off[n_docs])) return fail(B2T_ERR_INVALID, "%s: null argument", fn);
  int rc;
  if (dq && (rc = make_dense_req(spec, dq))) return rc;
  if (doc_off[0] != 0) return fail(B2T_ERR_INVALID, "doc_off[0] must be 0");
  for (uint32_t d = 0; d < n_docs; ++d)  // the kernels index the buffer with these: a decreasing offset must never reach them
    if (doc_off[d + 1] < doc_off[d]) return fail(B2T_ERR_INVALID, "doc_off must be non-decreasing (document %u)", d);
  std::unique_lock<std::mutex> prof(e->prof_mu, std::defer_lock);
  SetLease lease(e);
  if (e->profiling) prof.lock();
  CU(cudaSetDevice(e->device));
  return run(*lease.ss);
}

extern "C" int b2t_encode_batch(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, uint32_t flags,
                                b2t_result** out) {
  return host_call("b2t_encode_batch", e, bytes, doc_off, n_docs, out, nullptr, nullptr,
                   [&](b2t_engine::SlotSet& ss) { return host_encode(e, ss, bytes, doc_off, n_docs, flags, out); });
}

extern "C" int b2t_encode_batch_dense(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, const b2t_dense_spec* spec,
                                      b2t_result** out) {
  DenseReq dq;
  return host_call("b2t_encode_batch_dense", e, bytes, doc_off, n_docs, out, spec, &dq,
                   [&](b2t_engine::SlotSet& ss) { return host_encode(e, ss, bytes, doc_off, n_docs, 0u, out, &dq); });
}

// PreTokenizer seam: runs K0/K1 and expands the split bitmaps into (start, end) pairs.  The expansion of the bitmap
// into the pair list is output formatting and happens on the host (this is an inspection API, not the hot path).
static int pre_tokenize(b2t_engine* e, b2t_engine::SlotSet& ss, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, b2t_result** out) {
  const uint64_t n = doc_off[n_docs];
  Workspace& ws = ss.slot[0];
  int rc;
  if ((rc = slot_init(ws)) || (rc = ws.bytes.ensure(n + 64)) || (rc = ws.doc_off.ensure(((size_t)n_docs + 1) * 8))) return rc;
  if (n) CU(cudaMemcpyAsync(ws.bytes.p, bytes, n, cudaMemcpyHostToDevice, ws.stream));
  CU(cudaMemcpyAsync(ws.doc_off.p, doc_off, ((size_t)n_docs + 1) * 8, cudaMemcpyHostToDevice, ws.stream));
  ws.req = Request{ws.bytes.as<uint8_t>(), (int64_t)n, ws.doc_off.as<uint64_t>(), n_docs, B2T_NO_ADDED_TOKENS, RUN_PRETOK, nullptr};  // (a PreTokenizer knows no added tokens)
  if ((rc = run_device_pipeline(e, ws, ws.stream))) return rc;
  const uint64_t n_eff = (uint64_t)ws.batch.n;   // bytes the kernels ran on (n + inserted prefix spaces)
  const size_t n_words = n_eff / 32 + 2;
  std::vector<uint32_t> sb(n_words), db(n_words, 0u);
  CU(cudaMemcpyAsync(sb.data(), ws.start_bits.p, n_words * 4, cudaMemcpyDeviceToHost, ws.stream));
  if (pretok_drops_whitespace(e->pretok)) CU(cudaMemcpyAsync(db.data(), ws.drop_bits.p, n_words * 4, cudaMemcpyDeviceToHost, ws.stream));
  CU(cudaStreamSynchronize(ws.stream));
  b2t_result* r = pool_get(e);
  r->eng = e; r->on_device = 0; r->n_docs = n_docs;
  auto bit = [](const std::vector<uint32_t>& v, uint64_t p) { return (v[p >> 5] >> (p & 31)) & 1u; };
  uint64_t count = 0;
  for (uint64_t p = 0; p < n_eff; ++p) count += bit(sb, p) && !bit(db, p);
  if ((rc = r->h_offsets.ensure((count + 1) * 8, false)) || (rc = r->h_row_ptr.ensure(((size_t)n_docs + 1) * 8, false))) { pool_put(e, r); return rc; }
  uint32_t* off = r->h_offsets.as<uint32_t>();
  uint64_t* rp = r->h_row_ptr.as<uint64_t>();
  uint64_t k = 0, shift = 0;
  for (uint32_t d = 0; d < n_docs; ++d) {
    rp[d] = k;
    const uint64_t len = doc_off[d + 1] - doc_off[d];
    const bool pre = e->add_prefix_space && len > 0 && bytes[doc_off[d]] != ' ';
    const uint64_t dstart = doc_off[d] + shift;          // start of the document in the (re-packed) device batch
    const uint64_t end = dstart + len + (pre ? 1 : 0);
    uint64_t first_len = 1;                               // bytes of the first original character
    if (pre) { while (first_len < len && (bytes[doc_off[d] + first_len] & 0xC0) == 0x80) ++first_len; }
    uint64_t p = dstart;
    while (p < end) {
      uint64_t q = p + 1;
      while (q < end && !bit(sb, q)) ++q;
      if (!bit(db, p)) {
        uint64_t a = p - dstart, b = q - dstart;
        if (pre) { b = (b == 1) ? first_len : b - 1; a = a ? a - 1 : 0; }  // the inserted space is aligned to the first character
        off[2 * k] = (uint32_t)a; off[2 * k + 1] = (uint32_t)b; ++k;
      }
      p = q;
    }
    if (pre) ++shift;
  }
  rp[n_docs] = k;
  r->n_tokens = k; r->ids = nullptr; r->word_ids = nullptr; r->offsets = off; r->row_ptr = rp;
  *out = r;
  return B2T_OK;
}

extern "C" int b2t_pre_tokenize_batch(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, b2t_result** out) {
  return host_call("b2t_pre_tokenize_batch", e, bytes, doc_off, n_docs, out, nullptr, nullptr,
                   [&](b2t_engine::SlotSet& ss) { return pre_tokenize(e, ss, bytes, doc_off, n_docs, out); });
}

// ------------------------------------------------------------------------------------------------ results
extern "C" uint64_t b2t_result_n_tokens(const b2t_result* r) { return r ? r->n_tokens : 0; }
extern "C" uint32_t b2t_result_n_docs(const b2t_result* r) { return r ? r->n_docs : 0; }
extern "C" int b2t_result_on_device(const b2t_result* r) { return r ? r->on_device : 0; }
extern "C" const uint32_t* b2t_result_ids(const b2t_result* r) { return r ? r->ids : nullptr; }
extern "C" const uint32_t* b2t_result_offsets(const b2t_result* r) { return r ? r->offsets : nullptr; }
extern "C" const uint32_t* b2t_result_word_ids(const b2t_result* r) { return r ? r->word_ids : nullptr; }
extern "C" const uint64_t* b2t_result_row_ptr(const b2t_result* r) { return r ? r->row_ptr : nullptr; }
extern "C" uint32_t b2t_result_dense_length(const b2t_result* r) { return r ? r->dense_len : 0; }
extern "C" const uint32_t* b2t_result_dense_ids(const b2t_result* r) { return r ? r->dense_ids : nullptr; }
extern "C" const uint8_t* b2t_result_attention_mask(const b2t_result* r) { return r ? r->dense_mask : nullptr; }
extern "C" const uint32_t* b2t_result_row_lengths(const b2t_result* r) { return r ? r->row_len : nullptr; }
extern "C" void b2t_result_free(b2t_result* r) {
  if (!r) return;
  if (r->on_device || !r->eng) { delete r; return; }
  b2t_engine* e = r->eng;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->pool.size() < 4) e->pool.emplace_back(r);
  else { cudaSetDevice(e->device); delete r; }
}

extern "C" int b2t_host_alloc(size_t bytes, void** out) {
  if (!out) return fail(B2T_ERR_INVALID, "null argument");
  CU(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
  return B2T_OK;
}
extern "C" void b2t_host_free(void* p) { if (p) cudaFreeHost(p); }
