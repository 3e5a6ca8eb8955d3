// tests/native/pretok_emul.cpp -- runs the pre-tokenization scan (tokenizers_b200/csrc/pretok_logic.cuh) on the CPU,
// chunk by chunk, composed as pretok_lean_kernel / pretok_stream_kernel compose it.  TEST INFRASTRUCTURE: lets the CPU
// test suite fuzz the bit-parallel classification and boundary algebra against the oracle without a GPU.  Not linked
// into the product library.
#include <cstdint>
#include <cstring>
#include <vector>
#include "../../tokenizers_b200/csrc/pretok_logic.cuh"

using namespace b2t;

// Classification (bit planes, certain classes, table look-ups, fill, spill-in from the previous chunk), then per kind:
//   GPT-2 / Whitespace / Bert / no regex: the 32-bit algebra, contraction overflow into the next chunk, finalize_gpt2
//     with the next chunk's first bits;
//   Llama-3: the window algebra on [previous | own | next] and, when it reports `slow`, the slow path with chunk
//     classes computed standalone from the bytes, as the kernel's slow path computes them.
// gave_back: chunks whose straddling multi-byte space finalize_gpt2 gave back; slow: chunks that took the slow path.
template <int KIND>
static void emul(const uint8_t* bytes, uint64_t n, const uint64_t* doc_off, uint32_t n_docs, const uint32_t* cls_tbl,
                 uint32_t* start_bits, uint32_t* drop_bits, uint64_t* gave_back, uint64_t* slow) {
  const int64_t n_chunks = (int64_t)(n / CHUNK) + 1;
  std::vector<uint32_t> DS(n_chunks + 2, 0);
  for (uint32_t d = 0; d <= n_docs; ++d) DS[doc_off[d] / 32] |= 1u << (doc_off[d] % 32);
  auto at = [&](int64_t p) -> uint32_t { return (p >= 0 && (uint64_t)p < n) ? bytes[p] : 0u; };
  auto at4 = [&](int64_t p) -> uint32_t { return at(p) | (at(p + 1) << 8) | (at(p + 2) << 16) | (at(p + 3) << 24); };
  auto words = [&](int64_t c, uint32_t w[8]) { for (int j = 0; j < 8; ++j) w[j] = at4(c * 32 + j * 4); };
  auto valid = [&](int64_t c) -> uint32_t {
    const int64_t base = c * 32;
    return base + 32 <= (int64_t)n ? 0xFFFFFFFFu : (base >= (int64_t)n ? 0u : (0xFFFFFFFFu >> (32 - (int)((int64_t)n - base))));
  };
  std::vector<FastCls> M(n_chunks + 1);
  std::vector<PrevTop> PT(n_chunks + 1);
  FastCls prev;
  std::memset(&prev, 0, sizeof(prev));
  for (int64_t c = 0; c <= n_chunks; ++c) {
    uint32_t w[8], b[8];
    words(c, w);
    bitslice32(w, b);
    FastCls m = classify_planes<KIND>(b, valid(c));
    if (m.unc) resolve_uncertain(m, at4, c * 32, cls_tbl);
    fill_own(m);
    PrevTop pt; pt.L = prev.L; pt.N = prev.N; pt.S = prev.S; pt.SP = prev.SP;
    if (m.cont & 1u) spill_in(m, pt.L, pt.N, pt.S);
    M[c] = m; PT[c] = pt; prev = m;
  }
  Overflow ov_in; ov_in.bits = 0u;
  uint64_t n_gave_back = 0, n_slow = 0;
  for (int64_t c = 0; c < n_chunks; ++c) {
    const FastCls& m = M[c];
    const FastCls& x = M[c + 1];
    uint32_t start, drop = 0u;
    if (KIND == PT_LLAMA3) {
      FastCls p;
      if (c > 0) p = M[c - 1]; else std::memset(&p, 0, sizeof(p));
      Window w;
      w.lead = win(p.lead, m.lead, x.lead); w.L = win(p.L, m.L, x.L); w.N = win(p.N, m.N, x.N); w.S = win(p.S, m.S, x.S);
      w.SP = win(p.SP, m.SP, x.SP); w.NL = win(p.NL, m.NL, x.NL); w.AP = win(p.AP, m.AP, x.AP);
      w.DS = win(c > 0 ? DS[c - 1] : 0u, DS[c], DS[c + 1]);
      LlamaCarry cy; cy.n_count_before_window = 0; cy.zone_before_window = false; cy.tail_after_window = false;
      const BoundaryOut r = boundaries_llama3(w, c * 32 - 16, at4, cy);
      start = r.start;
      if (r.slow) {
        ++n_slow;
        auto masks = [&](int64_t k) {
          uint32_t wk[8];
          words(k, wk);
          return classify_standalone<KIND>(wk, valid(k), k * 32, at4, cls_tbl);
        };
        auto ds = [&](int64_t k) -> uint32_t { return (k >= 0 && k < n_chunks) ? DS[k] : 0u; };
        start = llama3_slow_path(w, c, n_chunks, masks, ds, at4);
      }
    } else {
      FastOut o;
      if (KIND == PT_GPT2) o = fast_gpt2(m, PT[c], DS[c], DS[c + 1], c * 32, at4);
      else if (KIND == PT_WHITESPACE) o = fast_whitespace(m, PT[c], DS[c]);
      else if (KIND == PT_BERT) o = fast_bert(m, PT[c], DS[c]);
      else { o.start = DS[c] & m.lead; o.drop = 0; o.ov.bits = 0; }
      start = apply_overflow(o.start, m.lead, ov_in);
      drop = o.drop;
      if (KIND == PT_GPT2) {
        const uint32_t before = start;
        start = finalize_gpt2(start, m.lead, m.S >> 31, x.lead & 15u, x.S & 15u, DS[c + 1]);
        if (start != before && (m.hi >> 31)) ++n_gave_back;   // counts the straddling multi-byte spaces that were given back
      }
      ov_in = o.ov;
    }
    start_bits[c] = start;
    if (drop_bits) drop_bits[c] = drop;
  }
  if (gave_back) *gave_back = n_gave_back;
  if (slow) *slow = n_slow;
}

extern "C" int b2t_emul_pretok(int kind, const uint8_t* bytes, uint64_t n, const uint64_t* doc_off, uint32_t n_docs,
                               const uint32_t* cls_tbl, uint32_t* start_bits, uint32_t* drop_bits, uint64_t* gave_back,
                               uint64_t* slow) {
  switch (kind) {
    case PT_GPT2: emul<PT_GPT2>(bytes, n, doc_off, n_docs, cls_tbl, start_bits, drop_bits, gave_back, slow); return 0;
    case PT_LLAMA3: emul<PT_LLAMA3>(bytes, n, doc_off, n_docs, cls_tbl, start_bits, drop_bits, gave_back, slow); return 0;
    case PT_WHITESPACE: emul<PT_WHITESPACE>(bytes, n, doc_off, n_docs, cls_tbl, start_bits, drop_bits, gave_back, slow); return 0;
    case PT_NOREGEX: emul<PT_NOREGEX>(bytes, n, doc_off, n_docs, cls_tbl, start_bits, drop_bits, gave_back, slow); return 0;
    case PT_BERT: emul<PT_BERT>(bytes, n, doc_off, n_docs, cls_tbl, start_bits, drop_bits, gave_back, slow); return 0;
    default: return 1;
  }
}

// Every code point >= 0x80 through classify_planes at every alignment of interest: wherever the boolean classifier
// claims a class (no `unc` bit), the claim must equal the class table.  cls8: 0x110000 bytes, one class per code point.
// Returns the number of wrong claims; *first_bad = first offending code point; *n_certain = code points with a claim.
template <int KIND>
static uint64_t check_claims(const uint8_t* cls8, uint32_t* first_bad, uint64_t* n_certain) {
  uint64_t bad = 0, certain = 0;
  for (uint32_t cp = 0x80; cp < 0x110000; ++cp) {
    if (cp >= 0xD800 && cp < 0xE000) continue;
    uint8_t enc[4]; int len;
    if (cp < 0x800) { enc[0] = 0xC0 | (cp >> 6); enc[1] = 0x80 | (cp & 63); len = 2; }
    else if (cp < 0x10000) { enc[0] = 0xE0 | (cp >> 12); enc[1] = 0x80 | ((cp >> 6) & 63); enc[2] = 0x80 | (cp & 63); len = 3; }
    else { enc[0] = 0xF0 | (cp >> 18); enc[1] = 0x80 | ((cp >> 12) & 63); enc[2] = 0x80 | ((cp >> 6) & 63); enc[3] = 0x80 | (cp & 63); len = 4; }
    bool any = false;
    for (int pos : {0, 7, 28, 29, 30, 31}) {
      uint8_t buf[32];
      std::memset(buf, 'a', 32);
      for (int k = 0; k < len && pos + k < 32; ++k) buf[pos + k] = enc[k];
      uint32_t w[8], b[8];
      std::memcpy(w, buf, 32);
      bitslice32(w, b);
      FastCls m = classify_planes<KIND>(b, 0xFFFFFFFFu);
      const uint32_t bit = 1u << pos;
      if (m.unc & bit) continue;
      any = true;
      const uint32_t claimed = (m.L & bit) ? CLS_L : (m.N & bit) ? CLS_N : (m.S & bit) ? CLS_S : CLS_O;
      if (claimed != cls8[cp]) { if (!bad) *first_bad = cp; ++bad; }
    }
    certain += any;
  }
  *n_certain = certain;
  return bad;
}
extern "C" uint64_t b2t_emul_check_claims(int kind, const uint8_t* cls8, uint32_t* first_bad, uint64_t* n_certain) {
  if (kind == PT_WHITESPACE) return check_claims<PT_WHITESPACE>(cls8, first_bad, n_certain);
  if (kind == PT_LLAMA3) return check_claims<PT_LLAMA3>(cls8, first_bad, n_certain);
  return check_claims<PT_GPT2>(cls8, first_bad, n_certain);
}

// bitslice32 against the definition
extern "C" int b2t_emul_check_bitslice(uint64_t seed, int rounds) {
  uint64_t s = seed;
  for (int r = 0; r < rounds; ++r) {
    uint8_t buf[32];
    for (int i = 0; i < 32; ++i) { s = s * 6364136223846793005ull + 1442695040888963407ull; buf[i] = (uint8_t)(s >> 56); }
    uint32_t w[8], b[8];
    std::memcpy(w, buf, 32);
    bitslice32(w, b);
    for (int j = 0; j < 8; ++j) {
      uint32_t e = 0;
      for (int p = 0; p < 32; ++p) e |= (uint32_t)((buf[p] >> j) & 1u) << p;
      if (e != b[j]) return 1;
    }
  }
  return 0;
}
