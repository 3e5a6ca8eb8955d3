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
#include "decode_kernels.cuh"
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
    if (kind == NORM_STRING) { src = nh.pool.data() + (e >> 8); len = (e >> 2) & NORM_LEN_MASK; }
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

// Dense mode request (b2t_encode_batch_dense*, b2t_encode_pairs_dense*): the device-side spec plus how L is chosen.
struct DenseReq {
  DenseSpec S;                  // single sequences (docs_per_row 1)
  PairDenseSpec P;              // pairs (docs_per_row 2): documents 2p and 2p + 1 make row p
  uint32_t docs_per_row = 1;
  bool batch_longest = false;   // padding strategy BatchLongest: L = longest row of the batch (after pad_to_multiple_of)
  uint32_t multiple = 0;        // pad_to_multiple_of
  bool want_mask = false;
  // overflowing parts (B2T_DENSE_OVERFLOW): rows per input are known after the count pass; offset rows (B2T_DENSE_OFFSETS)
  bool overflow = false, offsets = false;
  uint32_t stride = 0, type_oa = 0, type_ob = 0;
  // row metadata (B2T_DENSE_TRIM_OFFSETS .. B2T_DENSE_WORD_IDS): the META instantiations of the row kernels
  bool trim = false, aps = false, special_mask = false, seq_ids = false, word_ids = false;
  bool pairs() const { return docs_per_row == 2; }
  bool meta() const { return trim || special_mask || seq_ids || word_ids; }
  uint32_t& L() { return pairs() ? P.L : S.L; }
  uint32_t L() const { return pairs() ? P.L : S.L; }
};

// The outputs of dense mode: the bytes of one element, one element per cell of the [R, L] rows or per row, and what in
// the request asks for it.  The workspace, the pinned result and the result's views hold one buffer per output.
enum DenseOut { OUT_IDS, OUT_MASK, OUT_LEN, OUT_TYPE, OUT_SAMPLE, OUT_OFF, OUT_SPECIAL, OUT_SEQ, OUT_WORD, N_DENSE_OUT };
struct DenseOutput {
  uint32_t elem;
  bool per_row;
  bool (*wanted)(const DenseReq&);
};
constexpr DenseOutput DENSE_OUT[N_DENSE_OUT] = {
    {4, false, [](const DenseReq&) { return true; }},               // ids
    {1, false, [](const DenseReq& q) { return q.want_mask; }},      // attention mask
    {4, true, [](const DenseReq&) { return true; }},                // row lengths
    {1, false, [](const DenseReq& q) { return q.pairs(); }},        // type ids
    {4, true, [](const DenseReq& q) { return q.overflow; }},        // row sample: the input of each row
    {8, false, [](const DenseReq& q) { return q.offsets; }},        // offset rows: (start, end)
    {1, false, [](const DenseReq& q) { return q.special_mask; }},   // special-tokens mask
    {1, false, [](const DenseReq& q) { return q.seq_ids; }},        // sequence ids
    {4, false, [](const DenseReq& q) { return q.word_ids; }},       // word ids
};
// the bytes of one row of output k
static size_t dense_row_bytes(int k, uint32_t L) { return DENSE_OUT[k].per_row ? DENSE_OUT[k].elem : (size_t)DENSE_OUT[k].elem * L; }

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
  DevBuf dense[N_DENSE_OUT];           // dense rows (dense_kernels.cuh), one buffer per DenseOut
  DevBuf row_count, row_lexcl, row_bsum, row_base;   // overflow rows: the count pass, its scan and each input's first row
  // BertNormalizer pre-pass (norm_kernels.cuh): the normalized batch and what maps its tokens back to the original
  DevBuf nrm_doc_bits, nrm_pfd, nrm_page_out, nrm_page_chars, nrm_lexcl_o, nrm_bsum_o, nrm_lexcl_c, nrm_bsum_c, nrm_tot, nrm_bytes, nrm_src_char, nrm_doc_off, nrm_doc_char0;
  bool norm_active = false;
  DevBuf cand0, cand1, cand_any, hard_bits, inner_bits, added_bits, added_head, added_pool;
  uint32_t added_cap = 0;  // added-token extraction (added_kernels.cuh)
  DevBuf pfx_bytes, pfx_doc_off, pfx_local, pfx_block, prefix_bits, pfx_total;  // add_prefix_space re-pack (prefix_kernels.cuh)
  // decoding (decode_kernels.cuh): staged rows (host path), D1's counts and scan, D2's text, D3's lossy counts, scan and text
  DevBuf dec_ids, dec_row_ptr, dec_row_len, dec_count, dec_lexcl, dec_bsum, dec_text, dec_off, dec_lcount, dec_lexcl2, dec_bsum2, dec_text2, dec_off2;
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
  struct Views {   // what the accessors return: all null / 0 in a result the pool hands out
    const uint32_t* ids = nullptr; const uint32_t* offsets = nullptr; const uint32_t* word_ids = nullptr; const uint64_t* row_ptr = nullptr;
    // dense mode (b2t_encode_batch_dense*, b2t_encode_pairs_dense*): [n_rows, dense_len] rows instead of the CSR (n_docs =
    // pairs for a pair result; n_rows = n_docs without overflowing parts)
    uint32_t dense_len = 0, n_rows = 0;
    const void* dense[N_DENSE_OUT] = {};
    // decoding (b2t_decode_batch*): text of n_docs rows
    const uint8_t* text = nullptr; const uint64_t* text_off = nullptr;
  } view;
  PinBuf h_ids, h_offsets, h_word_ids, h_row_ptr;  // host results own pinned memory (returned to the engine pool on free)
  PinBuf h_dense[N_DENSE_OUT];
  PinBuf h_text, h_text_off;
};

// Publishes the dense views of a finished result: output k at buf[k] (the workspace's or the pinned result's buffers)
// where the request asks for it.
template <class Buf>
static void set_dense_views(b2t_result* r, const DenseReq& dq, uint32_t n_rows, const Buf (&buf)[N_DENSE_OUT]) {
  r->view.dense_len = dq.L(); r->view.n_rows = n_rows;
  for (int k = 0; k < N_DENSE_OUT; ++k) r->view.dense[k] = DENSE_OUT[k].wanted(dq) ? buf[k].p : nullptr;
}

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
  // offset trimming in dense rows (BPE engines): per vocabulary id / per added token (dense_kernels.cuh DenseMeta)
  DevBuf d_trim_vocab, d_trim_added;
  uint32_t n_trim_added = 0;
  int trim_ready = 0, added_both = 0;   // added_both: an added token has lstrip and rstrip (the rows may refuse it)
  // decoding: the model's vocabulary as the engine received it (the decoder table is built from it and the decoder spec)
  std::vector<uint8_t> vocab_bytes;
  std::vector<uint32_t> vocab_off, vocab_ids;
  int dec_on = 0, dec_kind = 0;   // b2t_engine_set_decoder
  DecodeTable dec{};
  DevBuf d_dec_ent, d_dec_pool;
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
  for (int i = 0; i < N_MODEL_LAYOUTS; ++i) {
    cudaFuncSetAttribute(model_kernel<MODEL_BPE>(i), cudaFuncAttributePreferredSharedMemoryCarveout, 86);
    cudaFuncSetAttribute(model_kernel<MODEL_WORDPIECE>(i), cudaFuncAttributePreferredSharedMemoryCarveout, 86);
  }
  if (cfg->model == B2T_MODEL_BPE) {   // (the ByteLevel pre-tokenizers: the only ones BPE runs behind)
    if ((rc = upload(e->d_trim_vocab, vocab_trim_counts(cfg->n_vocab, cfg->vocab_bytes, cfg->vocab_off, cfg->vocab_ids)))) return rc;
    e->trim_ready = 1;
  }
  e->vocab_bytes.assign(cfg->vocab_bytes, cfg->vocab_bytes + cfg->vocab_off[cfg->n_vocab]);
  e->vocab_off.assign(cfg->vocab_off, cfg->vocab_off + cfg->n_vocab + 1);
  e->vocab_ids.assign(cfg->vocab_ids, cfg->vocab_ids + cfg->n_vocab);
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
  uint32_t max_all;      // dense mode with overflowing parts: longest of all rows
  unsigned long long rows;   // dense mode with overflowing parts: rows of the batch
  uint32_t stride_m;     // ERR_STRIDE: the max_len the reference would panic on
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
// A spec read at the caller's struct_size: the current size, or the size before the fields from `stride` on were appended
// (those read as 0).  false = neither.
template <class Spec>
static bool read_spec(const Spec* sp, Spec* out) {
  constexpr size_t head = offsetof(Spec, stride), head_size = (head + 7) & ~(size_t)7;   // the old sizeof, tail padding included
  if (sp->struct_size != sizeof(Spec) && sp->struct_size != head_size) return false;
  memset(out, 0, sizeof(Spec));
  memcpy(out, sp, sp->struct_size == sizeof(Spec) ? sizeof(Spec) : head);
  return true;
}
static_assert(offsetof(b2t_dense_spec, stride) == 60 && offsetof(b2t_pair_dense_spec, stride) == 60, "the specs' first layout was 64 bytes");

static int dense_flags(uint32_t flags, uint32_t stride, DenseReq* dq) {
  constexpr uint32_t known = B2T_DENSE_OVERFLOW | B2T_DENSE_OFFSETS | B2T_DENSE_TRIM_OFFSETS | B2T_DENSE_TRIM_PREFIX_SPACE | B2T_DENSE_SPECIAL_MASK |
                             B2T_DENSE_SEQUENCE_IDS | B2T_DENSE_WORD_IDS;
  if (flags & ~known) return fail(B2T_ERR_INVALID, "unknown dense_flags 0x%x", flags);
  dq->overflow = (flags & B2T_DENSE_OVERFLOW) != 0; dq->offsets = (flags & B2T_DENSE_OFFSETS) != 0;
  dq->stride = dq->overflow ? stride : 0u;
  dq->trim = (flags & B2T_DENSE_TRIM_OFFSETS) != 0; dq->aps = (flags & B2T_DENSE_TRIM_PREFIX_SPACE) != 0;
  if (dq->trim && !dq->offsets) return fail(B2T_ERR_INVALID, "B2T_DENSE_TRIM_OFFSETS trims offset rows: it needs B2T_DENSE_OFFSETS");
  if (dq->aps && !dq->trim) return fail(B2T_ERR_INVALID, "B2T_DENSE_TRIM_PREFIX_SPACE is a rule of offset trimming: it needs B2T_DENSE_TRIM_OFFSETS");
  dq->special_mask = (flags & B2T_DENSE_SPECIAL_MASK) != 0; dq->seq_ids = (flags & B2T_DENSE_SEQUENCE_IDS) != 0;
  dq->word_ids = (flags & B2T_DENSE_WORD_IDS) != 0;
  return B2T_OK;
}

// What a dense request asks of the engine: trimming needs its vocabulary counts (BPE); the CSR flags the run needs for
// offset rows, word ids and, behind trimming, the added-token marks
static int dense_engine_flags(const b2t_engine* e, const DenseReq& dq, uint32_t* flags) {
  if (dq.trim && !e->trim_ready) return fail(B2T_ERR_UNSUPPORTED, "offset trimming (B2T_DENSE_TRIM_OFFSETS) needs a BPE engine behind a ByteLevel pre-tokenizer");
  *flags = (dq.offsets ? B2T_WANT_OFFSETS : 0u) | (dq.word_ids ? B2T_WANT_WORD_IDS : 0u) | (dq.trim && e->has_added ? B2T_FLAG_ADDED_IDS : 0u);
  return B2T_OK;
}

// The tail both spec readers share, after the template: the length budget left beside its n_special tokens (*budget) and
// how rows are padded.  dq->docs_per_row is set.
template <class Spec>
static int dense_length(const Spec* sp, uint32_t n_special, uint32_t* budget, DenseReq* dq) {
  // tokenizer/mod.rs:1272-1283: the sequence (or the pair) is truncated to max_length - n_added_tokens
  if (sp->max_length && sp->max_length < n_special) return fail(B2T_ERR_INVALID, "max_length %u is smaller than the %u special tokens of the template", sp->max_length, n_special);
  *budget = sp->max_length ? sp->max_length - n_special : DENSE_NO_LIMIT;
  dq->batch_longest = sp->length == 0;
  dq->multiple = sp->pad_to_multiple_of;
  dq->L() = dq->batch_longest ? 0u : dense_round(sp->length, dq->multiple);
  dq->want_mask = sp->want_mask != 0;
  return B2T_OK;
}

// b2t_dense_spec -> DenseReq, checked
static int make_dense_req(const b2t_dense_spec* sp_in, DenseReq* dq) {
  if (!sp_in) return fail(B2T_ERR_INVALID, "dense spec is null");
  b2t_dense_spec spec;
  if (!read_spec(sp_in, &spec)) return fail(B2T_ERR_INVALID, "b2t_dense_spec: struct_size mismatch (%u != %zu)", sp_in->struct_size, sizeof(b2t_dense_spec));
  const b2t_dense_spec* sp = &spec;
  int rc;
  if ((rc = dense_flags(sp->dense_flags, sp->stride, dq))) return rc;
  if (sp->n_pre > (uint32_t)DENSE_MAX_SPECIAL || sp->n_post > (uint32_t)DENSE_MAX_SPECIAL)
    return fail(B2T_ERR_UNSUPPORTED, "templates with more than %d special tokens on one side are not supported", DENSE_MAX_SPECIAL);
  if ((sp->n_pre && !sp->pre_ids) || (sp->n_post && !sp->post_ids)) return fail(B2T_ERR_INVALID, "dense spec: null special-token list");
  memset(&dq->S, 0, sizeof(dq->S));
  dq->S.pad_id = sp->pad_id; dq->S.n_pre = sp->n_pre; dq->S.n_post = sp->n_post;
  dq->S.trunc_left = sp->truncate_left ? 1 : 0; dq->S.pad_left = sp->pad_left ? 1 : 0;
  for (uint32_t i = 0; i < sp->n_pre; ++i) dq->S.pre[i] = sp->pre_ids[i];
  for (uint32_t i = 0; i < sp->n_post; ++i) dq->S.post[i] = sp->post_ids[i];
  return dense_length(sp, sp->n_pre + sp->n_post, &dq->S.keep_max, dq);
}
// b2t_pair_dense_spec -> DenseReq (pairs), checked: the piece list is split into pre X mid Y post
static int make_dense_req(const b2t_pair_dense_spec* sp_in, DenseReq* dq) {
  if (!sp_in) return fail(B2T_ERR_INVALID, "pair dense spec is null");
  b2t_pair_dense_spec spec;
  if (!read_spec(sp_in, &spec))
    return fail(B2T_ERR_INVALID, "b2t_pair_dense_spec: struct_size mismatch (%u != %zu)", sp_in->struct_size, sizeof(b2t_pair_dense_spec));
  const b2t_pair_dense_spec* sp = &spec;
  int rc;
  if ((rc = dense_flags(sp->dense_flags, sp->stride, dq))) return rc;
  if (dq->overflow && (sp->overflow_type_a > 255 || sp->overflow_type_b > 255))
    return fail(B2T_ERR_UNSUPPORTED, "overflow type ids %u / %u: type ids above 255 are not supported", sp->overflow_type_a, sp->overflow_type_b);
  dq->type_oa = sp->overflow_type_a; dq->type_ob = sp->overflow_type_b;
  if (sp->n_pieces && (!sp->piece_ids || !sp->piece_types)) return fail(B2T_ERR_INVALID, "pair dense spec: null piece list");
  if (sp->strategy < B2T_TRUNC_LONGEST_FIRST || sp->strategy > B2T_TRUNC_ONLY_SECOND) return fail(B2T_ERR_INVALID, "unknown truncation strategy %d", sp->strategy);
  if (sp->pad_type_id > 255) return fail(B2T_ERR_UNSUPPORTED, "pad type id %u: type ids above 255 are not supported", sp->pad_type_id);
  PairDenseSpec& P = dq->P;
  memset(&P, 0, sizeof(P));
  uint32_t n_seg[3] = {0, 0, 0}, seg = 0, n_a = 0, n_b = 0;
  for (uint32_t i = 0; i < sp->n_pieces; ++i) {
    const uint32_t id = sp->piece_ids[i], ty = sp->piece_types[i];
    if (ty > 255) return fail(B2T_ERR_UNSUPPORTED, "template type id %u: type ids above 255 are not supported", ty);
    if (id == B2T_PIECE_A || id == B2T_PIECE_B) {
      const bool x = seg == 0;   // the first sequence piece is X
      if (id == B2T_PIECE_A) ++n_a; else ++n_b;
      if (x) P.b_first = id == B2T_PIECE_B;
      (x ? P.type_x : P.type_y) = ty;
      ++seg;
      continue;
    }
    if (id >= (1u << 20)) return fail(B2T_ERR_UNSUPPORTED, "template token id %u: ids of 2^20 and above are not supported", id);
    if (seg > 2 || n_seg[seg] >= (uint32_t)DENSE_MAX_SPECIAL)
      return fail(B2T_ERR_UNSUPPORTED, "pair templates with more than %d special tokens before, between or after the sequences are not supported", DENSE_MAX_SPECIAL);
    P.special[seg * DENSE_MAX_SPECIAL + n_seg[seg]++] = id | ty << 24;
  }
  if (n_a != 1 || n_b != 1) return fail(B2T_ERR_INVALID, "a pair template holds sequence A and sequence B exactly once each");
  // pre, mid, post back to back, as the kernel indexes them
  for (uint32_t i = 0; i < n_seg[1]; ++i) P.special[n_seg[0] + i] = P.special[DENSE_MAX_SPECIAL + i];
  for (uint32_t i = 0; i < n_seg[2]; ++i) P.special[n_seg[0] + n_seg[1] + i] = P.special[2 * DENSE_MAX_SPECIAL + i];
  P.n_pre = n_seg[0]; P.n_mid = n_seg[1]; P.n_post = n_seg[2];
  P.strategy = (uint32_t)sp->strategy;
  P.pad_id = sp->pad_id; P.pad_type = sp->pad_type_id;
  P.trunc_left = sp->truncate_left ? 1 : 0; P.pad_left = sp->pad_left ? 1 : 0;
  dq->docs_per_row = 2;
  return dense_length(sp, P.n_pre + P.n_mid + P.n_post, &P.budget, dq);
}

// output k of the workspace's dense rows, null where the request does not ask for it
template <class T>
static T* dense_out(const Workspace& ws, const DenseReq& dq, DenseOut k) { return DENSE_OUT[k].wanted(dq) ? ws.dense[k].as<T>() : nullptr; }

// <OVER>: rows of overflowing parts (O's row fields); <OFFS>: offset rows (O's offset fields); <META>: row metadata (M)
template <bool OVER, bool OFFS, bool META>
static void launch_rows(Workspace& ws, uint32_t n_rows, const DenseReq& dq, const DenseOverflow& O, const DenseMeta& M, cudaStream_t st) {
  const unsigned grid = (unsigned)(((uint64_t)n_rows * 32 + 255) / 256);
  if (dq.pairs())
    dense_pair_rows_kernel<OVER, OFFS, META><<<grid, 256, 0, st>>>(ws.ids.as<uint32_t>(), ws.row_ptr.as<uint64_t>(), n_rows, dq.P, dense_out<uint32_t>(ws, dq, OUT_IDS),
                                                                   dense_out<uint8_t>(ws, dq, OUT_TYPE), dense_out<uint8_t>(ws, dq, OUT_MASK),
                                                                   dense_out<uint32_t>(ws, dq, OUT_LEN), O, M);
  else
    dense_rows_kernel<OVER, OFFS, META><<<grid, 256, 0, st>>>(ws.ids.as<uint32_t>(), ws.row_ptr.as<uint64_t>(), n_rows, dq.S, dense_out<uint32_t>(ws, dq, OUT_IDS),
                                                              dense_out<uint8_t>(ws, dq, OUT_MASK), dense_out<uint32_t>(ws, dq, OUT_LEN), nullptr, O, M);
}
using LaunchRows = void (*)(Workspace&, uint32_t, const DenseReq&, const DenseOverflow&, const DenseMeta&, cudaStream_t);
constexpr LaunchRows LAUNCH_ROWS[2][2][2] = {   // [OVER][OFFS][META]
    {{launch_rows<false, false, false>, launch_rows<false, false, true>}, {launch_rows<false, true, false>, launch_rows<false, true, true>}},
    {{launch_rows<true, false, false>, launch_rows<true, false, true>}, {launch_rows<true, true, false>, launch_rows<true, true, true>}}};

// CSR of the workspace -> dense rows in ws.dense (asynchronous on st).  n_inputs = documents / docs_per_row; n_rows =
// n_inputs, or with overflowing parts the rows the count pass found (the host has read them), whose row sample entries
// are the inputs' indices + sample_base.
static int launch_dense(b2t_engine* e, Workspace& ws, uint32_t n_inputs, uint32_t n_rows, const DenseReq& dq, cudaStream_t st, uint32_t sample_base = 0) {
  int rc;
  for (int k = 0; k < N_DENSE_OUT; ++k)
    if (DENSE_OUT[k].wanted(dq) && (rc = ws.dense[k].ensure(n_rows * dense_row_bytes(k, dq.L()) + 16))) return rc;
  DenseOverflow O{};
  if (dq.overflow) {
    if ((rc = ws.row_base.ensure((size_t)n_inputs * 4 + 16))) return rc;
    if (n_inputs)
      dense_row_sample_kernel<<<(unsigned)(((uint64_t)n_inputs * 32 + 255) / 256), 256, 0, st>>>(
          ws.row_count.as<uint32_t>(), ws.row_lexcl.as<unsigned long long>(), ws.row_bsum.as<unsigned long long>(), TSCAN, n_inputs, sample_base,
          ws.row_base.as<uint32_t>(), ws.dense[OUT_SAMPLE].as<uint32_t>());
    e->last_launches++;
    rec(e, st, "dense_row_sample");   // (from the end of dense_count: includes the host's read of the row count)
    const bool b_first = dq.pairs() && dq.P.b_first;
    O.row_sample = ws.dense[OUT_SAMPLE].as<uint32_t>(); O.row_base = ws.row_base.as<uint32_t>(); O.sample_base = sample_base; O.stride = dq.stride;
    O.type_ox = b_first ? dq.type_ob : dq.type_oa; O.type_oy = b_first ? dq.type_oa : dq.type_ob;
  }
  if (dq.offsets) { O.offsets = ws.offsets.as<uint2>(); O.out_off = ws.dense[OUT_OFF].as<uint2>(); }
  DenseMeta M{};
  if (dq.meta())
    M = DenseMeta{dq.trim ? e->d_trim_vocab.as<uint32_t>() : nullptr, e->has_added ? e->d_trim_added.as<AddedTrim>() : nullptr,
                  e->has_added ? e->n_trim_added : 0u, dq.aps ? 1u : 0u, dq.word_ids ? ws.word_ids.as<uint32_t>() : nullptr,
                  dense_out<uint8_t>(ws, dq, OUT_SPECIAL), dense_out<int8_t>(ws, dq, OUT_SEQ), dense_out<uint32_t>(ws, dq, OUT_WORD),
                  &ws.ctl.as<ctl_block>()->err};
  if (n_rows && dq.L()) LAUNCH_ROWS[dq.overflow][dq.offsets][dq.meta()](ws, n_rows, dq, O, M, st);
  e->last_launches++;
  if (dq.overflow) rec(e, st, dq.pairs() ? "dense_pair_rows_overflow" : "dense_rows_overflow");
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
// back at the end (N3 in finish_device); costs one small host sync for the size of the normalized batch.  Not for the
// PreTokenizer seam (RUN_PRETOK): a PreTokenizer splits the text it is given, and the seam's offsets index that text.
static int normalize(b2t_engine* e, Workspace& ws, Batch& b, uint32_t flags, cudaStream_t st) {
  ws.norm_active = false;
  if (!e->norm_on || ws.req.until == RUN_PRETOK || b.n == 0 || b.n_docs == 0) return B2T_OK;
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
    return fail(B2T_ERR_UNSUPPORTED, "the text holds a combining character that strip_accents keeps next to another combining character "
                "or a removed one: their canonical order (NFD) is not restated on the device");
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
static int model_and_count(b2t_engine* e, Workspace& ws, const Batch& b, uint32_t flags, bool added, cudaStream_t st) {
  const int64_t n_pages = b.n / PAGE + 1;
  // the page kernel's instance for what the call wants per token (behind the normalizer: byte offsets of the normalized
  // document, mapped back by norm_offsets_kernel)
  const bool offs = flags & B2T_WANT_OFFSETS;
  const unsigned lay = (offs ? L_OFFSETS : 0u) | ((flags & B2T_WANT_WORD_IDS) ? L_WORD_IDS : 0u) |
                       (offs && ((flags & B2T_OFFSETS_BYTES) || ws.norm_active) ? L_BYTE_OFFSETS : 0u) |
                       (offs && b.prefix_bits ? L_PREFIX : 0u) | (added && (flags & B2T_FLAG_ADDED_IDS) ? L_ADDED_IDS : 0u);
  const int li = model_layout_index(lay);
  if (li < 0) return fail(B2T_ERR_INVALID, "no page kernel for output layout %u", lay);
  ModelParams P;
  P.bytes = b.bytes; P.n = b.n;
  P.start_bits = ws.start_bits.as<uint32_t>(); P.drop_bits = ws.drop_bits.as<uint32_t>(); P.doc_bits = ws.doc_bits.as<uint32_t>();
  P.soft_bits = ws.soft_bits.as<uint32_t>(); P.page_soft = ws.page_soft.as<uint8_t>();
  P.page_carry = ws.page_carry.as<uint64_t>(); P.block_carry = ws.block_carry.as<uint64_t>(); P.page_first_doc = ws.page_first_doc.as<uint32_t>();
  P.doc_off = b.doc_off; P.n_docs = b.n_docs;
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
  P.t = e->dt;
  const ModelKernel k = e->model == B2T_MODEL_BPE ? model_kernel<MODEL_BPE>(li) : model_kernel<MODEL_WORDPIECE>(li);
  k<<<(unsigned)n_pages, MODEL_THREADS, 0, st>>>(P);
  rec(e, st, e->model == B2T_MODEL_BPE ? "bpe_tile" : "wordpiece_tile"); e->last_launches++;
  const int64_t n_tblk = (n_pages + TSCAN - 1) / TSCAN;
  tile_scan_block_kernel<<<(unsigned)n_tblk, TSCAN, 0, st>>>(ws.tile_count.as<uint32_t>(), ws.tile_lexcl.as<unsigned long long>(),
                                                           ws.tile_bsum.as<unsigned long long>(), n_pages);
  tile_scan_top_kernel<<<1, TSCAN, 0, st>>>(ws.tile_bsum.as<unsigned long long>(), n_tblk, &ctl->total);
  e->last_launches += 2;
  return B2T_OK;
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
    const uint32_t n_rows = n_docs / dq->docs_per_row;
    const PairDenseSpec& P = dq->P;
    if (n_rows && dq->pairs())
      pair_len_max_kernel<<<(n_rows + 255) / 256, 256, 0, st>>>(ws.row_ptr.as<uint64_t>(), n_rows, P.budget, P.strategy, P.n_pre + P.n_mid + P.n_post,
                                                              &ctl->max_row, &ctl->err);
    else if (n_rows)
      row_len_max_kernel<<<(n_rows + 255) / 256, 256, 0, st>>>(ws.row_ptr.as<uint64_t>(), n_rows, dq->S.keep_max, dq->S.n_pre + dq->S.n_post, &ctl->max_row);
    e->last_launches++;
    if (dq->overflow) {
      // the rows of every input and the longest of them; an exclusive scan of the counts gives each input's first row
      // (the rows themselves follow once the host has read the total)
      const uint32_t budget = dq->pairs() ? P.budget : dq->S.keep_max, n_special = dq->pairs() ? P.n_pre + P.n_mid + P.n_post : dq->S.n_pre + dq->S.n_post;
      const int64_t n_blk = ((int64_t)n_rows + TSCAN - 1) / TSCAN;
      if ((rc = ws.row_count.ensure((size_t)n_rows * 4 + 16)) || (rc = ws.row_lexcl.ensure((size_t)n_rows * 8 + 16)) ||
          (rc = ws.row_bsum.ensure((size_t)n_blk * 8 + 16)))
        return rc;
      if (n_rows) {
        dense_count_kernel<<<(n_rows + 255) / 256, 256, 0, st>>>(ws.row_ptr.as<uint64_t>(), n_rows, dq->pairs() ? 1u : 0u, budget, dq->pairs() ? P.strategy : 0u, dq->stride,
                                                               n_special, ws.row_count.as<uint32_t>(), &ctl->max_all, &ctl->err, &ctl->stride_m);
        tile_scan_block_kernel<<<(unsigned)n_blk, TSCAN, 0, st>>>(ws.row_count.as<uint32_t>(), ws.row_lexcl.as<unsigned long long>(),
                                                                 ws.row_bsum.as<unsigned long long>(), n_rows);
        tile_scan_top_kernel<<<1, TSCAN, 0, st>>>(ws.row_bsum.as<unsigned long long>(), n_blk, &ctl->rows);
        e->last_launches += 3;
      }
      rec(e, st, "dense_count");
    } else {
      if (!dq->batch_longest && (rc = launch_dense(e, ws, n_rows, n_rows, *dq, st))) return rc;
      rec(e, st, dq->pairs() ? "dense_pair_rows" : "dense_rows");
    }
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
    if ((rc = model_and_count(e, ws, b, q.flags, added, st)) || (rc = finish_tail(e, ws, st))) return rc;
  }
  CU(cudaGetLastError());
  return B2T_OK;
}

static int trim_ambiguous() {
  return fail(B2T_ERR_UNSUPPORTED, "offset trimming: an added token with both lstrip and rstrip absorbed whitespace, and its offsets do not tell "
              "on which side; trim_offsets is not available for this batch");
}

// Row kernels that run after the host has read the control block (overflowing parts, BatchLongest): an offset trimming
// that may meet an lstrip + rstrip added token reads the control block's error word again once they are done.
static int meta_check(b2t_engine* e, Workspace& ws, const DenseReq& dq, cudaStream_t st) {
  if (!dq.trim || !e->has_added || !e->added_both) return B2T_OK;
  ctl_block* h = ws.h_ctl.as<ctl_block>();
  CU(cudaMemcpyAsync(&h->err, &ws.ctl.as<ctl_block>()->err, 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (h->err & ERR_INTERNAL) return fail(B2T_ERR_CUDA, "internal error: a marked added-token id without an added token");
  return (h->err & ERR_TRIM_AMBIGUOUS) ? trim_ambiguous() : B2T_OK;
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
    if (!(c->lc.err & ERR_POOL_OVERFLOW)) {
      if (c->err & ERR_TRUNCATION) return fail(B2T_ERR_TRUNCATION, "Truncation error: Sequence to truncate too short to respect the provided max_length");
      if (c->err & ERR_STRIDE)
        return fail(B2T_ERR_TRUNCATION, "`stride` must be strictly less than `max_len=%u` (note that `max_len` may be shorter than the max length of the "
                    "original model, as it subtracts the number of special characters", c->stride_m);
      if (c->err & ERR_TRIM_AMBIGUOUS) return trim_ambiguous();
      return B2T_OK;
    }
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

// the spec argument of the entry points that are not dense
static const b2t_dense_spec* const NO_SPEC = nullptr;

// The device-resident entry points: argument checks (and in dense mode the spec -- b2t_dense_spec or b2t_pair_dense_spec --
// read into *dq), then the whole call under dev_mu on the engine's one device workspace, on the caller's stream or the
// engine's own.  `done(ws, st)` takes the finished run after the host has waited for it.
template <class Spec, class Done>
static int device_encode(const char* fn, b2t_engine* e, const void* out, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off,
                         uint32_t n_docs, uint32_t flags, RunUntil until, const Spec* spec, DenseReq* dq, void* stream, Done&& done) {
  if (!e || !out || !d_doc_off || (!d_bytes && n_bytes)) return fail(B2T_ERR_INVALID, "%s: null argument", fn);
  if (((uintptr_t)d_bytes & 15u) != 0) return fail(B2T_ERR_INVALID, "%s: d_bytes must be 16-byte aligned", fn);
  int rc;
  if (dq && (rc = make_dense_req(spec, dq))) return rc;
  if (dq && (rc = dense_engine_flags(e, *dq, &flags))) return rc;   // offset rows come from the CSR's offsets, word ids from its word ids
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
  return device_encode("b2t_encode_batch_device", e, out, d_bytes, n_bytes, d_doc_off, n_docs, flags, RUN_RESULT, NO_SPEC, nullptr, stream,
                       [&](Workspace& ws, cudaStream_t) -> int {
    b2t_result* r = new b2t_result();
    r->eng = e; r->on_device = 1; r->n_docs = n_docs;
    r->n_tokens = ws.h_ctl.as<ctl_block>()->total;
    r->view.ids = ws.ids.as<uint32_t>();
    r->view.offsets = (flags & B2T_WANT_OFFSETS) ? ws.offsets.as<uint32_t>() : nullptr;
    r->view.word_ids = (flags & B2T_WANT_WORD_IDS) ? ws.word_ids.as<uint32_t>() : nullptr;
    r->view.row_ptr = ws.row_ptr.as<uint64_t>();
    *out = r;
    return B2T_OK;
  });
}

extern "C" int b2t_encode_batch_device_begin(b2t_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off,
                                             uint32_t n_docs, uint32_t flags, void* stream, uint64_t* n_tokens) {
  return device_encode("b2t_encode_batch_device_begin", e, n_tokens, d_bytes, n_bytes, d_doc_off, n_docs, flags, RUN_COUNT, NO_SPEC, nullptr, stream,
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
  e->has_added = 0; e->added_both = 0; e->n_trim_added = 0;
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
  // offset trimming in dense rows: per token, by ascending id, its char count and leading / trailing whitespace-or-U+0120
  // counts, all-whitespace and its lstrip / rstrip flags (dense_kernels.cuh added_trim_counts)
  std::vector<AddedTrim> trim;
  for (int s2 = 0; s2 < 2; ++s2)
    for (uint32_t i : order[s2]) {
      uint32_t chars, lead, trail;
      space_counts(bytes + off[i], off[i + 1] - off[i], cls.data(), &chars, &lead, &trail);
      const bool l = (flags[i] & B2T_ADDED_LSTRIP) != 0, r = (flags[i] & B2T_ADDED_RSTRIP) != 0;
      trim.push_back(AddedTrim{ids[i], chars, std::min(lead, 0xFFFFu) | std::min(trail, 0xFFFFu) << 16,
                               (lead == chars ? TRIM_ALL_SPACE : 0u) | (l ? TRIM_LSTRIP : 0u) | (r ? TRIM_RSTRIP : 0u)});
      if (l && r) e->added_both = 1;
    }
  std::stable_sort(trim.begin(), trim.end(), [](const AddedTrim& a, const AddedTrim& b) { return a.id < b.id; });
  if ((rc = upload(e->d_trim_added, trim))) return rc;
  e->n_trim_added = (uint32_t)trim.size();
  e->has_added = 1;
  return B2T_OK;
}

// ------------------------------------------------------------------------------------------------ dense mode
// After a dense run with overflowing parts: the rows it makes (*n_rows; `before` rows precede them in the result) and
// whether they all fit L
static int overflow_rows(const ctl_block* c, uint64_t before, uint32_t L, uint32_t* n_rows) {
  if (before + c->rows >= (1ull << 31))
    return fail(B2T_ERR_TOO_LARGE, "the batch makes %llu dense rows or more: at most 2^31 - 1 fit one result", (unsigned long long)(before + c->rows));
  if (c->max_all > L)
    return fail(B2T_ERR_INVALID, "an overflowing row of %u tokens does not fit the dense length %u (the reference returns a longer, unpadded row here)", c->max_all, L);
  *n_rows = (uint32_t)c->rows;
  return B2T_OK;
}

// After the host has read the control block of a dense run of n_in inputs: L under BatchLongest, or the check that every
// row fits a fixed L; with overflowing parts the rows the run makes (`before` rows of the result precede them, the
// first input is sample_base); then the row kernels that had to wait for either (a fixed L without overflowing parts:
// queued with the run), asynchronous on st.  `room(*n_rows)` runs before they are queued: the host path makes room for
// the rows in its pinned result there.
template <class Room>
static int dense_after_count(b2t_engine* e, Workspace& ws, DenseReq& dq, uint32_t n_in, uint64_t before, uint32_t sample_base, cudaStream_t st,
                             uint32_t* n_rows, Room&& room) {
  const ctl_block* c = ws.h_ctl.as<ctl_block>();
  int rc;
  if (dq.batch_longest) dq.L() = dense_round(c->max_row, dq.multiple);
  else if (c->max_row > dq.L())
    return fail(B2T_ERR_INVALID, "a row of %u tokens does not fit the dense length %u: enable truncation (the reference returns a longer row here)", c->max_row, dq.L());
  *n_rows = n_in;
  if (dq.overflow && (rc = overflow_rows(c, before, dq.L(), n_rows))) return rc;
  if ((rc = room(*n_rows))) return rc;
  if ((dq.batch_longest || dq.overflow) && ((rc = launch_dense(e, ws, n_in, *n_rows, dq, st, sample_base)) || (rc = meta_check(e, ws, dq, st)))) return rc;
  return B2T_OK;
}

// the dense device entry points: the rows of n_docs / dq.docs_per_row inputs after the run, asynchronous on the stream
// like the CSR entry point's result
template <class Spec>
static int dense_device(const char* fn, b2t_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off, uint32_t n_docs,
                        const Spec* spec, void* stream, b2t_result** out) {
  DenseReq dq;
  return device_encode(fn, e, out, d_bytes, n_bytes, d_doc_off, n_docs, 0u, RUN_RESULT, spec, &dq, stream,
                       [&](Workspace& ws, cudaStream_t st) -> int {
    const uint32_t n_in = n_docs / dq.docs_per_row;
    uint32_t n_rows = 0;
    int rc2 = dense_after_count(e, ws, dq, n_in, 0, 0, st, &n_rows, [](uint32_t) { return B2T_OK; });
    if (rc2) return rc2;
    b2t_result* r = new b2t_result();
    r->eng = e; r->on_device = 1; r->n_docs = n_in;
    r->n_tokens = ws.h_ctl.as<ctl_block>()->total;
    set_dense_views(r, dq, n_rows, ws.dense);
    *out = r;
    return B2T_OK;
  });
}

extern "C" int b2t_encode_batch_dense_device(b2t_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off, uint32_t n_docs,
                                             const b2t_dense_spec* spec, void* stream, b2t_result** out) {
  return dense_device("b2t_encode_batch_dense_device", e, d_bytes, n_bytes, d_doc_off, n_docs, spec, stream, out);
}

// a batch of n_pairs pairs is a batch of 2 n_pairs documents
static int pair_docs(const char* fn, uint32_t n_pairs, uint32_t* n_docs) {
  if (n_pairs > UINT32_MAX / 2) return fail(B2T_ERR_TOO_LARGE, "%s: %u pairs are more than 2^32 - 1 documents", fn, n_pairs);
  *n_docs = 2 * n_pairs;
  return B2T_OK;
}

// Replaces TokenizerImpl::post_process for a batch of pairs (tokenizer/mod.rs:1265-1317), see include/b2t.h
extern "C" int b2t_encode_pairs_dense_device(b2t_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint64_t* d_doc_off, uint32_t n_pairs,
                                             const b2t_pair_dense_spec* spec, void* stream, b2t_result** out) {
  uint32_t n_docs = 0;
  int rc = pair_docs("b2t_encode_pairs_dense_device", n_pairs, &n_docs);
  return rc ? rc : dense_device("b2t_encode_pairs_dense_device", e, d_bytes, n_bytes, d_doc_off, n_docs, spec, stream, out);
}

// ------------------------------------------------------------------------------------------------ host pipeline
static b2t_result* pool_get(b2t_engine* e) {
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->pool.empty()) {
    b2t_result* r = e->pool.back().release(); e->pool.pop_back();
    r->view = {};
    return r;
  }
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

// Queues the copy of a chunk's dense rows (rows r0 .. r0 + nr - 1) into the pinned result, on the slot's stream.
static int queue_dense_copy(b2t_result* r, const Workspace& ws, uint32_t r0, uint32_t nr, const DenseReq& dq) {
  for (int k = 0; k < N_DENSE_OUT; ++k) {
    const size_t row = dense_row_bytes(k, dq.L());
    if (DENSE_OUT[k].wanted(dq) && nr && row)
      CU(cudaMemcpyAsync(r->h_dense[k].as<uint8_t>() + r0 * row, ws.dense[k].p, nr * row, cudaMemcpyDeviceToHost, ws.stream));
  }
  return B2T_OK;
}

static int host_encode(b2t_engine* e, b2t_engine::SlotSet& ss, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, uint32_t flags,
                       b2t_result** out, const DenseReq* dq_in = nullptr, uint32_t dq_flags = 0u) {
  const uint64_t total_bytes = doc_off[n_docs];
  // ---- split into chunks of whole documents
  std::vector<Chunk> chunks;
  uint64_t max_chunk = 0;
  DenseReq dq_local;
  DenseReq* dq = nullptr;
  if (dq_in) { dq_local = *dq_in; dq = &dq_local; flags = dq_flags; }   // (offset rows, word ids: from the CSR's)
  // BatchLongest padding needs every row length before the first row can be written: the batch runs as one chunk
  if (dq && dq->batch_longest && total_bytes + n_docs >= (1ull << 31))
    return fail(B2T_ERR_UNSUPPORTED, "dense output padded to the longest row needs the batch in one device pass (< 2^31 bytes); pad to a fixed length instead");
  const uint64_t chunk_bytes = (dq && dq->batch_longest) ? (1ull << 31) : (uint64_t)e->chunk_bytes;
  // chunks hold whole rows: per = documents per row (a pair's two documents stay in one chunk)
  const uint32_t per = dq ? dq->docs_per_row : 1u, n_rows = n_docs / per;
  {
    uint32_t d = 0;
    while (d < n_docs) {
      uint64_t limit = doc_off[d] + chunk_bytes;
      uint32_t d1 = (uint32_t)(std::upper_bound(doc_off + d + 1, doc_off + n_docs + 1, limit) - doc_off) - 1;
      d1 = d + (d1 - d) / per * per;
      if (d1 <= d) d1 = d + per;  // a single row larger than the chunk size
      if (doc_off[d1] - doc_off[d] >= (1ull << 31)) return fail(B2T_ERR_TOO_LARGE, per == 1 ? "document %u is larger than 2 GiB" : "pair %u is larger than 2 GiB", d / per);
      chunks.push_back({d, d1, doc_off[d], doc_off[d1], 0});
      max_chunk = std::max(max_chunk, doc_off[d1] - doc_off[d]);
      d = d1;
    }
    if (chunks.empty()) chunks.push_back({0, 0, 0, 0, 0});
  }
  b2t_result* r = pool_get(e);
  r->eng = e; r->on_device = 0; r->n_docs = dq ? n_rows : n_docs; r->n_tokens = 0;
  int rc;
  const bool want_off = !dq && (flags & B2T_WANT_OFFSETS) != 0, want_wid = (flags & B2T_WANT_WORD_IDS) != 0;
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
  // pinned rows: the whole batch's n_rows rows, or with overflowing parts a guess grown on demand (contents kept)
  uint64_t cap_rows = 0, row_total = 0;
  auto dense_host = [&](uint64_t rows, bool keep) -> int {
    int rc2;
    for (int k = 0; k < N_DENSE_OUT; ++k)
      if (DENSE_OUT[k].wanted(*dq) && (rc2 = r->h_dense[k].ensure(rows * dense_row_bytes(k, dq->L()) + 16, keep))) return rc2;
    cap_rows = rows;
    return B2T_OK;
  };
  if (dq) { if (!dq->batch_longest && (rc = dense_host(n_rows, false))) { pool_put(e, r); return rc; } }
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
      uint32_t nr = 0;
      auto room = [&](uint32_t rows) -> int {
        if (dq->overflow && row_total + rows > cap_rows) {
          // the chunk's rows go at the running row base; earlier chunks may still be copying into the old buffers: let
          // them land, then grow (contents are kept)
          for (auto& s : ss.slot) if (s.stream) CU(cudaStreamSynchronize(s.stream));
          return dense_host(std::max<uint64_t>((row_total + rows) * 2, (uint64_t)n_rows), true);
        }
        return (dq->batch_longest && !dq->overflow) ? dense_host(n_rows, false) : B2T_OK;   // (one chunk: L is known now)
      };
      if ((rc2 = dense_after_count(e, ws, *dq, (c.d1 - c.d0) / per, row_total, c.d0 / per, ws.stream, &nr, room))) return rc2;
      // (a fixed length without overflowing parts: the rows were queued for the copy right behind the kernels, see issue();
      // a rerun has replaced them)
      if ((dq->batch_longest || dq->overflow || reran) && (rc2 = queue_dense_copy(r, ws, (uint32_t)row_total, nr, *dq))) return rc2;
      row_total += nr;
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
    if (dq && !dq->batch_longest && !dq->overflow && (rc2 = queue_dense_copy(r, ws, c.d0 / per, nd / per, *dq))) return rc2;
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
    if (n_docs == 0 && dq->batch_longest) dq->L() = 0;
    r->n_tokens = tok_base;
    set_dense_views(r, *dq, (uint32_t)row_total, r->h_dense);
  } else {
    // chunk-relative row_ptr -> batch-relative (host fix-up: one addition per document)
    uint64_t* rp = r->h_row_ptr.as<uint64_t>();
    for (size_t ci = 1; ci < nc; ++ci) {
      const Chunk& c = chunks[ci];
      const uint32_t hi = (ci + 1 == nc) ? c.d1 : c.d1 - 1;
      for (uint32_t d = c.d0; d <= hi; ++d) rp[d] += c.tok_base;
    }
    r->n_tokens = tok_base;
    r->view.ids = r->h_ids.as<uint32_t>();
    r->view.offsets = want_off ? r->h_offsets.as<uint32_t>() : nullptr;
    r->view.word_ids = want_wid ? r->h_word_ids.as<uint32_t>() : nullptr;
    r->view.row_ptr = rp;
  }
  *out = r;
  return B2T_OK;
}

// The host-buffer entry points: argument checks (and in dense mode the spec, read into *dq), then `run(slot set)` on a slot
// set of the call's own -- and, while per-kernel profiling is on, on the whole engine (the event records are one per engine).
template <class Spec, class Run>
static int host_call(const char* fn, b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, b2t_result** out,
                     const Spec* spec, DenseReq* dq, Run&& run) {
  if (!e || !out || !doc_off || (!bytes && doc_off[n_docs])) return fail(B2T_ERR_INVALID, "%s: null argument", fn);
  int rc;
  uint32_t dq_flags = 0;
  if (dq && (rc = make_dense_req(spec, dq))) return rc;
  if (dq && (rc = dense_engine_flags(e, *dq, &dq_flags))) return rc;
  if (doc_off[0] != 0) return fail(B2T_ERR_INVALID, "doc_off[0] must be 0");
  for (uint32_t d = 0; d < n_docs; ++d)  // the kernels index the buffer with these: a decreasing offset must never reach them
    if (doc_off[d + 1] < doc_off[d]) return fail(B2T_ERR_INVALID, "doc_off must be non-decreasing (document %u)", d);
  std::unique_lock<std::mutex> prof(e->prof_mu, std::defer_lock);
  SetLease lease(e);
  if (e->profiling) prof.lock();
  CU(cudaSetDevice(e->device));
  return run(*lease.ss, dq_flags);
}

extern "C" int b2t_encode_batch(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, uint32_t flags,
                                b2t_result** out) {
  return host_call("b2t_encode_batch", e, bytes, doc_off, n_docs, out, NO_SPEC, nullptr,
                   [&](b2t_engine::SlotSet& ss, uint32_t) { return host_encode(e, ss, bytes, doc_off, n_docs, flags, out); });
}

extern "C" int b2t_encode_batch_dense(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, const b2t_dense_spec* spec,
                                      b2t_result** out) {
  DenseReq dq;
  return host_call("b2t_encode_batch_dense", e, bytes, doc_off, n_docs, out, spec, &dq,
                   [&](b2t_engine::SlotSet& ss, uint32_t dq_flags) { return host_encode(e, ss, bytes, doc_off, n_docs, 0u, out, &dq, dq_flags); });
}

// Replaces TokenizerImpl::post_process for a batch of pairs (tokenizer/mod.rs:1265-1317), see include/b2t.h
extern "C" int b2t_encode_pairs_dense(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_pairs, const b2t_pair_dense_spec* spec,
                                      b2t_result** out) {
  DenseReq dq;
  uint32_t n_docs = 0;
  int rc = pair_docs("b2t_encode_pairs_dense", n_pairs, &n_docs);
  if (rc) return rc;
  return host_call("b2t_encode_pairs_dense", e, bytes, doc_off, n_docs, out, spec, &dq,
                   [&](b2t_engine::SlotSet& ss, uint32_t dq_flags) { return host_encode(e, ss, bytes, doc_off, n_docs, 0u, out, &dq, dq_flags); });
}

// PreTokenizer seam: runs K0/K1 on the text as given (neither the normalizer nor the added tokens apply) and expands the
// split bitmaps into (start, end) pairs.  The expansion of the bitmap into the pair list is output formatting and
// happens on the host (this is an inspection API, not the hot path).
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
  if ((rc = r->h_row_ptr.ensure(((size_t)n_docs + 1) * 8, false))) { pool_put(e, r); return rc; }
  auto bit = [](const std::vector<uint32_t>& v, uint64_t p) { return (v[p >> 5] >> (p & 31)) & 1u; };
  // one walk over each document's range of the batch the kernels ran on both counts the splits and writes them, so the
  // bitmaps are never read outside that batch and the pairs never outgrow their buffer
  std::vector<uint32_t> pairs;
  uint64_t* rp = r->h_row_ptr.as<uint64_t>();
  uint64_t shift = 0;
  for (uint32_t d = 0; d < n_docs; ++d) {
    rp[d] = pairs.size() / 2;
    const uint64_t len = doc_off[d + 1] - doc_off[d];
    const bool pre = e->add_prefix_space && len > 0 && bytes[doc_off[d]] != ' ';
    const uint64_t dstart = doc_off[d] + shift;          // start of the document in the (re-packed) device batch
    const uint64_t end = dstart + len + (pre ? 1 : 0);
    if (end > n_eff) {
      pool_put(e, r);
      return fail(B2T_ERR_CUDA, "internal error: document %u ends at byte %llu of a pre-tokenized batch of %llu bytes", d,
                  (unsigned long long)end, (unsigned long long)n_eff);
    }
    uint64_t first_len = 1;                               // bytes of the first original character
    if (pre) { while (first_len < len && (bytes[doc_off[d] + first_len] & 0xC0) == 0x80) ++first_len; }
    uint64_t p = dstart;
    while (p < end) {
      uint64_t q = p + 1;
      while (q < end && !bit(sb, q)) ++q;
      if (!bit(db, p)) {
        uint64_t a = p - dstart, b = q - dstart;
        if (pre) { b = (b == 1) ? first_len : b - 1; a = a ? a - 1 : 0; }  // the inserted space is aligned to the first character
        pairs.push_back((uint32_t)a); pairs.push_back((uint32_t)b);
      }
      p = q;
    }
    if (pre) ++shift;
  }
  const uint64_t k = pairs.size() / 2;
  rp[n_docs] = k;
  if ((rc = r->h_offsets.ensure((k + 1) * 8, false))) { pool_put(e, r); return rc; }
  uint32_t* off = r->h_offsets.as<uint32_t>();
  if (k) memcpy(off, pairs.data(), k * 8);
  r->n_tokens = k; r->view.offsets = off; r->view.row_ptr = rp;
  *out = r;
  return B2T_OK;
}

extern "C" int b2t_pre_tokenize_batch(b2t_engine* e, const uint8_t* bytes, const uint64_t* doc_off, uint32_t n_docs, b2t_result** out) {
  return host_call("b2t_pre_tokenize_batch", e, bytes, doc_off, n_docs, out, NO_SPEC, nullptr,
                   [&](b2t_engine::SlotSet& ss, uint32_t) { return pre_tokenize(e, ss, bytes, doc_off, n_docs, out); });
}

// ------------------------------------------------------------------------------------------------ decoding
// The decoder spec, checked, -> the decoder table of a vocabulary (host only)
static int decoder_table(const b2t_decoder_spec* sp, bool normalizer, uint32_t n_vocab, const uint8_t* vb, const uint32_t* vo, const uint32_t* vi,
                         DecoderHost* dh) {
  if (sp->struct_size != sizeof(b2t_decoder_spec)) return fail(B2T_ERR_INVALID, "b2t_decoder_spec: struct_size mismatch (%u != %zu)", sp->struct_size, sizeof(b2t_decoder_spec));
  if (sp->n_added && (!sp->added_bytes || !sp->added_off || !sp->added_ids || !sp->added_flags)) return fail(B2T_ERR_INVALID, "decoder spec: null added-token list");
  const std::string msg = build_decoder_table(sp->kind, sp->prefix, sp->cleanup != 0, normalizer, n_vocab, vb, vo, vi, sp->n_added, sp->added_bytes,
                                              sp->added_off, sp->added_ids, sp->added_flags, dh);
  return msg.empty() ? B2T_OK : fail(B2T_ERR_UNSUPPORTED, "%s", msg.c_str());
}

extern "C" int b2t_decoder_images(const b2t_config* cfg, const b2t_decoder_spec* spec, uint64_t* table, uint8_t* pool, uint32_t* n_ids, uint64_t* pool_bytes) {
  if (!cfg || !spec || !n_ids || !pool_bytes || !cfg->vocab_bytes || !cfg->vocab_off || !cfg->vocab_ids) return fail(B2T_ERR_INVALID, "b2t_decoder_images: null argument");
  DecoderHost dh;
  int rc = decoder_table(spec, (cfg->bert_normalizer & B2T_NORM_BERT) != 0, cfg->n_vocab, cfg->vocab_bytes, cfg->vocab_off, cfg->vocab_ids, &dh);
  if (rc) return rc;
  *n_ids = (uint32_t)dh.ent.size(); *pool_bytes = dh.pool.size();
  if (table) memcpy(table, dh.ent.data(), dh.ent.size() * 8);
  if (pool) memcpy(pool, dh.pool.data(), dh.pool.size());
  return B2T_OK;
}

extern "C" int b2t_engine_set_decoder(b2t_engine* e, const b2t_decoder_spec* spec) {
  if (!e) return fail(B2T_ERR_INVALID, "null engine");
  std::lock_guard<std::mutex> lk(e->dev_mu);
  e->dec_on = 0;
  if (!spec) return B2T_OK;
  DecoderHost dh;
  int rc = decoder_table(spec, e->norm_on != 0, (uint32_t)e->vocab_ids.size(), e->vocab_bytes.data(), e->vocab_off.data(), e->vocab_ids.data(), &dh);
  if (rc) return rc;
  CU(cudaSetDevice(e->device));
  if ((rc = upload(e->d_dec_ent, dh.ent)) || (rc = upload(e->d_dec_pool, dh.pool))) return rc;
  e->dec = DecodeTable{e->d_dec_ent.as<uint2>(), e->d_dec_pool.as<uint8_t>(), (uint32_t)dh.ent.size()};
  e->dec_kind = spec->kind;
  e->dec_on = 1;
  return B2T_OK;
}

// D1-D3 on rows resident on the device (R), on st: *text / *text_off point at the workspace's finished text of *n_text
// bytes.  Synchronises for the size of the text and, for ByteLevel, for whether the lossy rewrite has to run and then
// for the rewritten size.  The profiling records name the host's reads (*_read) apart from the kernels.
static int run_decode(b2t_engine* e, Workspace& ws, const DecodeRows& R, uint32_t flags, cudaStream_t st, const uint8_t** text, const uint64_t** text_off,
                      uint64_t* n_text) {
  const uint32_t n = R.n_rows, skip = (flags & B2T_DECODE_SKIP_SPECIAL) ? 1u : 0u;
  const bool lossy = e->dec_kind == B2T_DECODER_BYTELEVEL;
  const int64_t n_blk = ((int64_t)n + TSCAN - 1) / TSCAN;
  const unsigned grid = (unsigned)(((uint64_t)n * 32 + DEC_THREADS - 1) / DEC_THREADS);
  int rc;
  if ((rc = ws.ctl.ensure(sizeof(DecodeCtl))) || (rc = ws.h_ctl.ensure(sizeof(DecodeCtl), false)) || (rc = ws.dec_count.ensure((size_t)n * 4 + 16)) ||
      (rc = ws.dec_lexcl.ensure((size_t)n * 8 + 16)) || (rc = ws.dec_bsum.ensure((size_t)n_blk * 8 + 16)) || (rc = ws.dec_off.ensure(((size_t)n + 1) * 8)) ||
      (lossy && ((rc = ws.dec_lcount.ensure((size_t)n * 4 + 16)) || (rc = ws.dec_lexcl2.ensure((size_t)n * 8 + 16)) ||
                 (rc = ws.dec_bsum2.ensure((size_t)n_blk * 8 + 16)) || (rc = ws.dec_off2.ensure(((size_t)n + 1) * 8)))))
    return rc;
  DecodeCtl* ctl = ws.ctl.as<DecodeCtl>();
  DecodeCtl* h = ws.h_ctl.as<DecodeCtl>();
  CU(cudaMemsetAsync(ctl, 0, sizeof(DecodeCtl), st));
  CU(cudaMemsetAsync(ws.dec_off.p, 0, 8, st));   // (text_off[0] of an empty batch)
  rec(e, st, nullptr);
  e->last_launches = 0;
  if (n) {
    decode_count_kernel<<<grid, DEC_THREADS, 0, st>>>(e->dec, R, skip, ws.dec_count.as<uint32_t>(), ctl);
    tile_scan_block_kernel<<<(unsigned)n_blk, TSCAN, 0, st>>>(ws.dec_count.as<uint32_t>(), ws.dec_lexcl.as<unsigned long long>(), ws.dec_bsum.as<unsigned long long>(), n);
    tile_scan_top_kernel<<<1, TSCAN, 0, st>>>(ws.dec_bsum.as<unsigned long long>(), n_blk, &ctl->total);
    e->last_launches += 3;
  }
  rec(e, st, "decode_count");
  CU(cudaMemcpyAsync(h, ctl, sizeof(DecodeCtl), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));   // the size of the text
  if (h->err & DEC_ERR_ROWS) return fail(B2T_ERR_INVALID, "decode: row_ptr decreasing or a row outside [0, n_ids)");
  if (h->err & DEC_ERR_ROW_SIZE) return fail(B2T_ERR_TOO_LARGE, "decode: the text of a row reaches %llu bytes; split the row", (unsigned long long)DEC_MAX_ROW_TEXT);
  const uint64_t total = h->total;
  if ((rc = ws.dec_text.ensure(total + 16))) return rc;
  rec(e, st, "decode_size_read");   // (the host's read of the text size: not kernel time)
  if (n)
    decode_emit_kernel<<<grid, DEC_THREADS, 0, st>>>(e->dec, R, skip, ws.dec_count.as<uint32_t>(), ws.dec_lexcl.as<unsigned long long>(), ws.dec_bsum.as<unsigned long long>(),
                                                     TSCAN, ws.dec_text.as<uint8_t>(), ws.dec_off.as<uint64_t>(), lossy ? ws.dec_lcount.as<uint32_t>() : nullptr, ctl);
  e->last_launches++;
  rec(e, st, "decode_emit");
  *text = ws.dec_text.as<uint8_t>(); *text_off = ws.dec_off.as<uint64_t>(); *n_text = total;
  if (!lossy || !n) { CU(cudaGetLastError()); return B2T_OK; }
  CU(cudaMemcpyAsync(&h->bad, &ctl->bad, 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (!h->bad) return B2T_OK;   // valid UTF-8 throughout: the text is final
  rec(e, st, "decode_flag_read");   // (the host's read of D2's flag: not kernel time)
  // the scan of D2's lossy counts gives the rewritten text's exact size before its buffer is sized
  tile_scan_block_kernel<<<(unsigned)n_blk, TSCAN, 0, st>>>(ws.dec_lcount.as<uint32_t>(), ws.dec_lexcl2.as<unsigned long long>(), ws.dec_bsum2.as<unsigned long long>(), n);
  tile_scan_top_kernel<<<1, TSCAN, 0, st>>>(ws.dec_bsum2.as<unsigned long long>(), n_blk, &ctl->lossy);
  rec(e, st, "decode_lossy_scan");
  CU(cudaMemcpyAsync(&h->lossy, &ctl->lossy, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if ((rc = ws.dec_text2.ensure(h->lossy + 16))) return rc;
  rec(e, st, "decode_lossy_read");   // (the host's read of the rewritten size: not kernel time)
  decode_lossy_kernel<<<grid, DEC_THREADS, 0, st>>>(ws.dec_text.as<uint8_t>(), ws.dec_off.as<uint64_t>(), n, ws.dec_lcount.as<uint32_t>(), ws.dec_lexcl2.as<unsigned long long>(),
                                                    ws.dec_bsum2.as<unsigned long long>(), TSCAN, ws.dec_text2.as<uint8_t>(), ws.dec_off2.as<uint64_t>());
  e->last_launches += 3;
  rec(e, st, "decode_lossy");
  *text = ws.dec_text2.as<uint8_t>(); *text_off = ws.dec_off2.as<uint64_t>(); *n_text = h->lossy;
  CU(cudaGetLastError());
  return B2T_OK;
}

// argument checks shared by both decode entry points
static int decode_args(const char* fn, b2t_engine* e, const void* ids, uint64_t n_ids, const uint64_t* row_ptr, uint32_t flags, b2t_result** out) {
  if (!e || !out || !row_ptr || (!ids && n_ids)) return fail(B2T_ERR_INVALID, "%s: null argument", fn);
  if (flags & ~(uint32_t)B2T_DECODE_SKIP_SPECIAL) return fail(B2T_ERR_INVALID, "%s: unknown flags 0x%x", fn, flags);
  if (n_ids >= (1ull << 31)) return fail(B2T_ERR_TOO_LARGE, "%s: %llu ids exceed the per-call limit of 2^31 - 1; split the batch", fn, (unsigned long long)n_ids);
  if (!e->dec_on) return fail(B2T_ERR_INVALID, "%s: the engine has no decoder (b2t_engine_set_decoder)", fn);
  return B2T_OK;
}

extern "C" int b2t_decode_batch_device(b2t_engine* e, const uint32_t* d_ids, uint64_t n_ids, const uint64_t* d_row_ptr, const uint32_t* d_row_len,
                                       uint32_t n_rows, uint32_t flags, void* stream, b2t_result** out) {
  int rc = decode_args("b2t_decode_batch_device", e, d_ids, n_ids, d_row_ptr, flags, out);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(e->dev_mu);
  CU(cudaSetDevice(e->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : e->own_stream;
  Workspace& ws = e->dev_ws;
  const uint8_t* text; const uint64_t* text_off; uint64_t n_text;
  if ((rc = run_decode(e, ws, DecodeRows{d_ids, d_row_ptr, d_row_len, 0ull, n_ids, n_rows}, flags, st, &text, &text_off, &n_text))) return rc;
  b2t_result* r = new b2t_result();
  r->eng = e; r->on_device = 1; r->n_docs = n_rows; r->n_tokens = n_text;
  r->view.text = text; r->view.text_off = text_off;
  *out = r;
  return B2T_OK;
}

// The host entry point: chunks of whole rows (ids spanning at most chunk_bytes / 4; a larger row is a chunk of its own) on
// the slot set's workspaces in turn.  A chunk's text is copied into the pinned result on its slot's stream while the next
// chunk is staged and decoded on the next slot.  That is the only overlap: a chunk's own kernels wait for the host's reads
// of run_decode (the text size, and for ByteLevel the lossy flag), so the copies in, the kernels and the copies out of
// one chunk do not overlap each other as they do in the encode pipeline.
static int host_decode(b2t_engine* e, b2t_engine::SlotSet& ss, const uint32_t* ids, const uint64_t* row_ptr, const uint32_t* row_len, uint32_t n_rows,
                       uint32_t flags, b2t_result** out) {
  const uint64_t chunk_ids = std::max<uint64_t>(e->chunk_bytes / 4, 1);
  auto row_end = [&](uint32_t r) { return row_len ? row_ptr[r] + row_len[r] : row_ptr[r + 1]; };
  b2t_result* r = pool_get(e);
  r->eng = e; r->on_device = 0; r->n_docs = n_rows; r->n_tokens = 0;
  int rc;
  uint64_t cap = 0, text_base = 0;
  if ((rc = r->h_text_off.ensure(((size_t)n_rows + 1) * 8, false)) || (rc = r->h_text.ensure(16, false))) { pool_put(e, r); return rc; }
  cap = r->h_text.cap;
  uint64_t* toff = r->h_text_off.as<uint64_t>();
  struct DecChunk { uint32_t r0, r1; uint64_t base; };
  std::vector<DecChunk> chunks;
  rc = B2T_OK;
  for (uint32_t r0 = 0, ci = 0; r0 < n_rows && rc == B2T_OK; ++ci) {
    const uint64_t lo = row_ptr[r0];
    uint64_t hi = row_end(r0);
    uint32_t r1 = r0 + 1;
    while (r1 < n_rows && std::max(hi, row_end(r1)) - lo <= chunk_ids) hi = std::max(hi, row_end(r1++));
    Workspace& ws = ss.slot[ci % NSLOT];
    auto step = [&]() -> int {
      int rc2;
      if ((rc2 = slot_init(ws))) return rc2;
      CU(cudaStreamSynchronize(ws.stream));   // (its previous chunk's copies have landed)
      const uint32_t nr = r1 - r0;
      if ((rc2 = ws.dec_ids.ensure((hi - lo) * 4 + 16)) || (rc2 = ws.dec_row_ptr.ensure(((size_t)nr + 1) * 8)) ||
          (row_len && (rc2 = ws.dec_row_len.ensure((size_t)nr * 4 + 16))))
        return rc2;
      if (hi > lo) CU(cudaMemcpyAsync(ws.dec_ids.p, ids + lo, (hi - lo) * 4, cudaMemcpyHostToDevice, ws.stream));
      CU(cudaMemcpyAsync(ws.dec_row_ptr.p, row_ptr + r0, ((size_t)nr + (row_len ? 0 : 1)) * 8, cudaMemcpyHostToDevice, ws.stream));
      if (row_len) CU(cudaMemcpyAsync(ws.dec_row_len.p, row_len + r0, (size_t)nr * 4, cudaMemcpyHostToDevice, ws.stream));
      const uint8_t* text; const uint64_t* text_off; uint64_t n_text;
      if ((rc2 = run_decode(e, ws, DecodeRows{ws.dec_ids.as<uint32_t>(), ws.dec_row_ptr.as<uint64_t>(), row_len ? ws.dec_row_len.as<uint32_t>() : nullptr, lo, hi - lo, nr},
                            flags, ws.stream, &text, &text_off, &n_text)))
        return rc2;
      if (text_base + n_text > cap) {
        // earlier chunks may still be copying into the old buffer: let them land, then grow (contents are kept)
        for (auto& s : ss.slot) if (s.stream) CU(cudaStreamSynchronize(s.stream));
        if ((rc2 = r->h_text.ensure((text_base + n_text) * 2, true))) return rc2;
        cap = r->h_text.cap;
      }
      if (n_text) CU(cudaMemcpyAsync(r->h_text.as<uint8_t>() + text_base, text, n_text, cudaMemcpyDeviceToHost, ws.stream));
      CU(cudaMemcpyAsync(toff + r0, text_off, (size_t)nr * 8, cudaMemcpyDeviceToHost, ws.stream));
      chunks.push_back({r0, r1, text_base});
      text_base += n_text;
      return B2T_OK;
    };
    rc = step();
    r0 = r1;
  }
  for (auto& s : ss.slot) if (s.stream) cudaStreamSynchronize(s.stream);
  if (rc) { pool_put(e, r); return rc; }
  // chunk-relative offsets -> batch-relative
  for (const DecChunk& c : chunks)
    if (c.base) for (uint32_t k = c.r0; k < c.r1; ++k) toff[k] += c.base;
  toff[n_rows] = text_base;
  r->n_tokens = text_base;
  r->view.text = r->h_text.as<uint8_t>(); r->view.text_off = toff;
  *out = r;
  return B2T_OK;
}

extern "C" int b2t_decode_batch(b2t_engine* e, const uint32_t* ids, uint64_t n_ids, const uint64_t* row_ptr, const uint32_t* row_len, uint32_t n_rows,
                                uint32_t flags, b2t_result** out) {
  int rc = decode_args("b2t_decode_batch", e, ids, n_ids, row_ptr, flags, out);
  if (rc) return rc;
  for (uint32_t r = 0; r < n_rows; ++r) {   // the kernels index the id buffer with these
    if (r + 1 < n_rows && row_ptr[r + 1] < row_ptr[r]) return fail(B2T_ERR_INVALID, "b2t_decode_batch: row_ptr must be non-decreasing (row %u)", r);
    const uint64_t end = row_len ? row_ptr[r] + row_len[r] : row_ptr[r + 1];
    if (end < row_ptr[r] || end > n_ids) return fail(B2T_ERR_INVALID, "b2t_decode_batch: row %u lies outside [0, n_ids)", r);
  }
  std::unique_lock<std::mutex> prof(e->prof_mu, std::defer_lock);
  SetLease lease(e);
  if (e->profiling) prof.lock();
  CU(cudaSetDevice(e->device));
  return host_decode(e, *lease.ss, ids, row_ptr, row_len, n_rows, flags, out);
}

// ------------------------------------------------------------------------------------------------ results
extern "C" uint64_t b2t_result_n_tokens(const b2t_result* r) { return r ? r->n_tokens : 0; }
extern "C" uint32_t b2t_result_n_docs(const b2t_result* r) { return r ? r->n_docs : 0; }
extern "C" int b2t_result_on_device(const b2t_result* r) { return r ? r->on_device : 0; }
extern "C" const uint32_t* b2t_result_ids(const b2t_result* r) { return r ? r->view.ids : nullptr; }
extern "C" const uint32_t* b2t_result_offsets(const b2t_result* r) { return r ? r->view.offsets : nullptr; }
extern "C" const uint32_t* b2t_result_word_ids(const b2t_result* r) { return r ? r->view.word_ids : nullptr; }
extern "C" const uint64_t* b2t_result_row_ptr(const b2t_result* r) { return r ? r->view.row_ptr : nullptr; }
extern "C" uint32_t b2t_result_dense_length(const b2t_result* r) { return r ? r->view.dense_len : 0; }
extern "C" uint32_t b2t_result_dense_rows(const b2t_result* r) { return r ? r->view.n_rows : 0; }
template <class T>
static const T* dense_view(const b2t_result* r, DenseOut k) { return r ? static_cast<const T*>(r->view.dense[k]) : nullptr; }
extern "C" const uint32_t* b2t_result_dense_ids(const b2t_result* r) { return dense_view<uint32_t>(r, OUT_IDS); }
extern "C" const uint8_t* b2t_result_attention_mask(const b2t_result* r) { return dense_view<uint8_t>(r, OUT_MASK); }
extern "C" const uint32_t* b2t_result_row_lengths(const b2t_result* r) { return dense_view<uint32_t>(r, OUT_LEN); }
extern "C" const uint8_t* b2t_result_type_ids(const b2t_result* r) { return dense_view<uint8_t>(r, OUT_TYPE); }
extern "C" const uint32_t* b2t_result_row_sample(const b2t_result* r) { return dense_view<uint32_t>(r, OUT_SAMPLE); }
extern "C" const uint32_t* b2t_result_dense_offsets(const b2t_result* r) { return dense_view<uint32_t>(r, OUT_OFF); }
extern "C" const uint8_t* b2t_result_special_tokens_mask(const b2t_result* r) { return dense_view<uint8_t>(r, OUT_SPECIAL); }
extern "C" const int8_t* b2t_result_sequence_ids(const b2t_result* r) { return dense_view<int8_t>(r, OUT_SEQ); }
extern "C" const uint32_t* b2t_result_dense_word_ids(const b2t_result* r) { return dense_view<uint32_t>(r, OUT_WORD); }
extern "C" const uint8_t* b2t_result_text(const b2t_result* r) { return r ? r->view.text : nullptr; }
extern "C" const uint64_t* b2t_result_text_off(const b2t_result* r) { return r ? r->view.text_off : nullptr; }
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
