// pretok_logic.cuh -- the pre-tokenization scan as bit-parallel mask algebra (host + device).
//
// Replaces the regex split of the reference's pre-tokenizers on the encode_batch path:
//   pre_tokenizers/byte_level.rs:43-46,119-131   GPT-2 pattern, split Isolated        (PT_GPT2)
//   pre_tokenizers/split.rs:96-104 + the tiktoken pattern (bindings/python/benches/test_tiktoken.py:38),
//     followed by ByteLevel(use_regex=false)                                           (PT_LLAMA3)
//   pre_tokenizers/whitespace.rs:20-29           \w+|[^\w\s]+, Invert + Removed        (PT_WHITESPACE)
//
// The text is cut into 32-byte chunks.  Phase A (`classify_chunk`) turns a chunk into 32-bit class masks, one bit per
// byte, continuation bytes inheriting the class of their character.  Phase B (`boundaries_*`) builds 64-bit windows
// [16 B before | 32 B own | 16 B after] from the neighbours' masks and evaluates, for all 32 positions at once, whether a
// pre-token starts there.  The ordered-alternation / backtracking semantics of the regexes reduce to predicates over
// a bounded neighbourhood plus three run properties (digit position mod 3, leading-newline zone, newline-free tail)
// that are propagated with Kogge-Stone steps inside the window; runs that reach a window edge take a slow path.
// Everything here is pure so that tests/native/pretok_emul.cpp can run exactly this code on the CPU.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2T_HD __host__ __device__ __forceinline__
#else
#define B2T_HD inline
#endif

namespace b2t {

enum PretokKind { PT_GPT2 = 0, PT_LLAMA3 = 1, PT_WHITESPACE = 2, PT_NOREGEX = 3, PT_BERT = 4 };   // PT_BERT: pre_tokenizers/bert.rs:5-19
B2T_HD bool pretok_drops_whitespace(int kind) { return kind == PT_WHITESPACE || kind == PT_BERT; }
enum { CLS_O = 0, CLS_L = 1, CLS_N = 2, CLS_S = 3 };

constexpr int CHUNK = 32;         // bytes per thread-chunk
constexpr int PAGE = 2048;        // bytes per page (summary granularity, tile of the model kernels)
constexpr int PAGE_CHUNKS = PAGE / CHUNK;

struct ChunkMasks {
  uint32_t lead;  // byte starts a character
  uint32_t L, N, S;  // class of the character the byte belongs to (onig: \p{L} \p{N} \s ; rust: \w, -, \s)
  uint32_t SP, NL, AP;  // U+0020 ; \r or \n ; apostrophe
};

struct Window {
  uint64_t lead, L, N, S, SP, NL, AP, DS;
};

#if defined(__CUDA_ARCH__)
B2T_HD int popc32(uint32_t x) { return __popc(x); }
B2T_HD int popc64(uint64_t x) { return __popcll(x); }
B2T_HD int clz64(uint64_t x) { return __clzll((long long)x); }
B2T_HD int ctz64(uint64_t x) { return __ffsll((long long)x) - 1; }
B2T_HD int ctz32(uint32_t x) { return __ffs((int)x) - 1; }
#else
B2T_HD int popc32(uint32_t x) { return __builtin_popcount(x); }
B2T_HD int popc64(uint64_t x) { return __builtin_popcountll(x); }
B2T_HD int clz64(uint64_t x) { return x ? __builtin_clzll(x) : 64; }
B2T_HD int ctz64(uint64_t x) { return x ? __builtin_ctzll(x) : -1; }
B2T_HD int ctz32(uint32_t x) { return x ? __builtin_ctz(x) : -1; }
#endif

// 2 bits per code point, 16 code points per u32 word.
B2T_HD uint32_t class_of(const uint32_t* __restrict__ tbl, uint32_t cp) {
  if (cp >= 0x110000u) return CLS_O;
#if defined(__CUDA_ARCH__)
  uint32_t w = __ldg(tbl + (cp >> 4));
#else
  uint32_t w = tbl[cp >> 4];
#endif
  return (w >> ((cp & 15u) * 2u)) & 3u;
}

// ---------------------------------------------------------------------------------------------- phase A
// two "bit 7 per byte" flag words -> one byte: low nibble = flags of a (byte 0 -> bit 0), high nibble = flags of b
B2T_HD uint32_t movemask2(uint32_t a, uint32_t b) {
  uint32_t x = (a >> 7) | (b >> 3);
  return (x * 0x01020408u) >> 24;
}

// Decode the UTF-8 character whose lead byte is at p (valid UTF-8 assumed; bytes past `end` read as 0).
template <class ByteAt>
B2T_HD uint32_t decode_at(const ByteAt& at, int64_t p, int64_t end, int* len) {
  uint32_t b0 = at(p);
  if (b0 < 0x80u) { *len = 1; return b0; }
  uint32_t b1 = p + 1 < end ? at(p + 1) : 0u;
  if (b0 < 0xE0u) { *len = 2; return ((b0 & 31u) << 6) | (b1 & 63u); }
  uint32_t b2 = p + 2 < end ? at(p + 2) : 0u;
  if (b0 < 0xF0u) { *len = 3; return ((b0 & 15u) << 12) | ((b1 & 63u) << 6) | (b2 & 63u); }
  uint32_t b3 = p + 3 < end ? at(p + 3) : 0u;
  *len = 4;
  return ((b0 & 7u) << 18) | ((b1 & 63u) << 12) | ((b2 & 63u) << 6) | (b3 & 63u);
}

// ASCII half of phase A.  Bit-7-per-byte flags are computed with SWAR range checks (3 ops each) and transposed into
// 32-bit position masks two words at a time (movemask2 gives 8 mask bits per multiply).  Apostrophes and control
// characters are rare, so their masks are built in a second pass only when a cheap detector saw one.
// Outputs: m.L / m.N / m.S / m.SP / m.NL / m.AP for ASCII bytes only, *hi = non-ASCII bytes, *cont = continuation bytes.
// kind: PT_WHITESPACE uses the Rust-regex classes (\w on ASCII = [0-9A-Za-z_], N slot unused).
B2T_HD void ascii_masks(int kind, const uint32_t w[8], ChunkMasks& m, uint32_t* hi_out, uint32_t* cont_out) {
  const bool rust = kind == PT_WHITESPACE;
  uint32_t L = 0, N = 0, SP = 0, CT = 0, HI = 0, any_ctl = 0, any_ap = 0, any_hi = 0;
#pragma unroll
  for (int j = 0; j < 8; j += 2) {
    uint32_t fL[2], fN[2], fSP[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t x = w[j + h];
      const uint32_t asc = ~x & 0x80808080u;            // bit 7 set <=> ASCII byte
      const uint32_t w7 = x & 0x7F7F7F7Fu;
      const uint32_t t = w7 | 0x20202020u;
      uint32_t l = (t + 0x1F1F1F1Fu) & ~(t + 0x05050505u) & asc;             // 'a'..'z' after folding case
      uint32_t d = (w7 + 0x50505050u) & ~(w7 + 0x46464646u) & asc;           // '0'..'9'
      if (rust) { l |= d | ((w7 + 0x21212121u) & ~(w7 + 0x20202020u) & asc); d = 0u; }  // + '_' (0x5F)
      fL[h] = l; fN[h] = d;
      fSP[h] = (w7 + 0x60606060u) & ~(w7 + 0x5F5F5F5Fu) & asc;               // == 0x20
      any_ctl |= ~(w7 + 0x60606060u) & asc;                                   // < 0x20
      any_ap |= (w7 + 0x59595959u) & ~(w7 + 0x58585858u) & asc;              // == 0x27
      any_hi |= x;
    }
    const int sh = 4 * j;  // 8 mask bits per pair of words
    L |= movemask2(fL[0], fL[1]) << sh;
    if (!rust) N |= movemask2(fN[0], fN[1]) << sh;
    SP |= movemask2(fSP[0], fSP[1]) << sh;
  }
  if (any_hi & 0x80808080u) {  // non-ASCII bytes are present: positions of all of them and of the continuation bytes
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      const uint32_t x0 = w[j], x1 = w[j + 1];
      CT |= movemask2(x0 & ~(x0 << 1) & 0x80808080u, x1 & ~(x1 << 1) & 0x80808080u) << (4 * j);   // 10xxxxxx
      HI |= movemask2(x0 & 0x80808080u, x1 & 0x80808080u) << (4 * j);
    }
  }
  uint32_t S = SP, NL = 0, AP = 0;
  if (any_ctl) {  // \t \n \v \f \r are whitespace; \n and \r are the newlines of the tiktoken pattern
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      uint32_t a[2], b[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t x = w[j + h], asc = ~x & 0x80808080u, w7 = x & 0x7F7F7F7Fu;
        a[h] = (w7 + 0x77777777u) & ~(w7 + 0x72727272u) & asc;                // 9..13
        b[h] = 0u;
        if (kind == PT_LLAMA3)  // only the tiktoken pattern distinguishes newlines
          b[h] = (((w7 + 0x76767676u) & ~(w7 + 0x75757575u)) | ((w7 + 0x73737373u) & ~(w7 + 0x72727272u))) & asc;  // 10, 13
      }
      S |= movemask2(a[0], a[1]) << (4 * j);
      if (kind == PT_LLAMA3) NL |= movemask2(b[0], b[1]) << (4 * j);
    }
  }
  if (any_ap && !rust) {  // apostrophes only matter to the contraction alternatives of the ByteLevel / tiktoken patterns
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      uint32_t a[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t x = w[j + h], asc = ~x & 0x80808080u, w7 = x & 0x7F7F7F7Fu;
        a[h] = (w7 + 0x59595959u) & ~(w7 + 0x58585858u) & asc;
      }
      AP |= movemask2(a[0], a[1]) << (4 * j);
    }
  }
  m.L = L; m.N = N; m.S = S; m.SP = SP; m.NL = NL; m.AP = AP; m.lead = ~CT;
  *hi_out = HI; *cont_out = CT;
}

// Class and length of the (non-ASCII) character whose UTF-8 bytes are b0 b1 b2 b3 (valid UTF-8 assumed).
B2T_HD uint32_t decode_class(uint32_t b0, uint32_t b1, uint32_t b2, uint32_t b3, const uint32_t* __restrict__ cls_tbl, int* len) {
  uint32_t cp;
  if (b0 < 0xE0u) { *len = 2; cp = ((b0 & 31u) << 6) | (b1 & 63u); }
  else if (b0 < 0xF0u) { *len = 3; cp = ((b0 & 15u) << 12) | ((b1 & 63u) << 6) | (b2 & 63u); }
  else { *len = 4; cp = ((b0 & 7u) << 18) | ((b1 & 63u) << 12) | ((b2 & 63u) << 6) | (b3 & 63u); }
  return class_of(cls_tbl, cp);
}

// Classify the 32 bytes [base, base+32) of a buffer of n bytes, everything included (generic path: CPU emulation,
// halo chunks and slow paths on the device).  w[0..7] are the chunk's bytes as little-endian words (bytes at
// positions >= n must be zero).  `at(pos)` gives random access to any byte in [0, n).
template <class ByteAt>
B2T_HD ChunkMasks classify_chunk(const uint32_t w[8], int64_t base, int64_t n, const ByteAt& at,
                                 const uint32_t* __restrict__ cls_tbl, int kind) {
  ChunkMasks m;
  uint32_t hi_any, cont;
  ascii_masks(kind, w, m, &hi_any, &cont);
  if (hi_any) {
    // a character that starts before the chunk but owns its first bytes
    if (cont & 1u) {
      int back = 1;
      while (back < 3 && (at(base - back) & 0xC0u) == 0x80u) ++back;
      int len;
      const int64_t q = base - back;
      uint32_t c = decode_class(at(q), at(q + 1), at(q + 2), at(q + 3), cls_tbl, &len);
      int cover = len - back;  // bytes of this char inside the chunk
      if (cover > 0) {
        uint32_t bits = (1u << cover) - 1u;
        if (c == CLS_L) m.L |= bits; else if (c == CLS_N) m.N |= bits; else if (c == CLS_S) m.S |= bits;
      }
    }
    uint32_t todo = hi_any & ~cont;  // non-ASCII lead bytes inside the chunk
    while (todo) {
      int p = ctz32(todo);
      todo &= todo - 1u;
      int len;
      const int64_t q = base + p;
      uint32_t c = decode_class(at(q), at(q + 1), at(q + 2), at(q + 3), cls_tbl, &len);
      uint32_t bits = ((1u << len) - 1u) << p;  // bits past 31 fall off: the next chunk redoes them
      if (c == CLS_L) m.L |= bits; else if (c == CLS_N) m.N |= bits; else if (c == CLS_S) m.S |= bits;
    }
  }
  // bytes at or past n: no class, no lead
  if (base + CHUNK > n) {
    uint32_t valid = (n <= base) ? 0u : (0xFFFFFFFFu >> (32 - (int)(n - base)));
    m.lead &= valid; m.L &= valid; m.N &= valid; m.S &= valid; m.SP &= valid; m.NL &= valid; m.AP &= valid;
  }
  return m;
}

// ---------------------------------------------------------------------------------------------- phase B helpers
B2T_HD uint64_t win(uint32_t prev, uint32_t own, uint32_t next) {
  return (uint64_t)(prev >> 16) | ((uint64_t)own << 16) | ((uint64_t)(next & 0xFFFFu) << 48);
}
constexpr uint64_t OWN = 0x0000FFFFFFFF0000ull;

// forward (towards higher positions) propagation of `seed` through positions allowed by `into`
// (position j may receive from j-1 iff into[j])
B2T_HD uint64_t prop_fwd(uint64_t seed, uint64_t into) {
  uint64_t p = seed, m = into;
  p |= (p << 1) & m;  m &= m << 1;
  p |= (p << 2) & m;  m &= m << 2;
  p |= (p << 4) & m;  m &= m << 4;
  p |= (p << 8) & m;  m &= m << 8;
  p |= (p << 16) & m; m &= m << 16;
  p |= (p << 32) & m;
  return p;
}
// backward propagation: position j may receive from j+1 iff into[j]
B2T_HD uint64_t prop_bwd(uint64_t seed, uint64_t into) {
  uint64_t p = seed, m = into;
  p |= (p >> 1) & m;  m &= m >> 1;
  p |= (p >> 2) & m;  m &= m >> 2;
  p |= (p >> 4) & m;  m &= m >> 4;
  p |= (p >> 8) & m;  m &= m >> 8;
  p |= (p >> 16) & m; m &= m >> 16;
  p |= (p >> 32) & m;
  return p;
}
// flag on a lead byte -> flag on the lead byte of the NEXT character (chars are <= 4 bytes)
B2T_HD uint64_t to_next_lead(uint64_t x, uint64_t lead) {
  uint64_t r, c;
  c = x << 1;            r = c & lead;  c &= ~lead;
  c <<= 1;               r |= c & lead; c &= ~lead;
  c <<= 1;               r |= c & lead; c &= ~lead;
  c <<= 1;               r |= c & lead;
  return r;
}
// For whitespace characters (<= 3 bytes): lead bytes of chars whose LAST byte carries flag m.
B2T_HD uint64_t last_byte_flag_to_lead(uint64_t m, uint64_t lead) {
  uint64_t c1 = ~lead >> 1;          // byte i+1 is a continuation byte
  uint64_t c2 = c1 & (~lead >> 2);   // bytes i+1, i+2 are continuation bytes
  return lead & ((m & ~c1) | ((m >> 1) & c1 & ~c2) | ((m >> 2) & c2));
}

struct BoundaryOut {
  uint32_t start;  // pre-token (split) starts among the chunk's 32 positions
  uint32_t drop;   // PT_WHITESPACE: starts of splits that the reference removes (whitespace)
  uint32_t slow;   // bit0: a run reaches a window edge, the caller must use the slow path for this chunk
};

// Contraction lengths for the apostrophe at window position a (needs raw bytes): 0 = none, 2 = 's etc, 3 = 're etc.
// Returned length is in BYTES after... i.e. the match is [a, a+len).  icase also folds U+017F to 's' (2 bytes => len 3).
template <class ByteAt, class Pos>
B2T_HD int contraction_len(const ByteAt& at, Pos pos, Pos doc_end_hint, bool icase) {
  // bytes past the end of the buffer read as 0 through `at`
  (void)doc_end_hint;
  uint32_t a = at(pos + 1), b = at(pos + 2);
  if (icase) {
    if (a == 0xC5u && b == 0xBFu) return 3;  // 'ſ
    if (a >= 'A' && a <= 'Z') a += 32;
    if (b >= 'A' && b <= 'Z') b += 32;
  }
  if (a == 's' || a == 't' || a == 'm' || a == 'd') return 2;
  if ((a == 'r' || a == 'v') && b == 'e') return 3;
  if (a == 'l' && b == 'l') return 3;
  return 0;
}

// Apply the contraction rules to `start` (window coordinates).  cand = apostrophes that sit at a match start.
template <class ByteAt>
B2T_HD uint64_t apply_contractions(uint64_t start, uint64_t cand, const Window& w, int64_t win_base, const ByteAt& at,
                                   bool icase, uint64_t* contr_start_out) {
  uint64_t cs = 0;
  // only apostrophes in window bits [12, 48) can influence own bits [16, 48)
  uint64_t todo = cand & 0x0000FFFFFFFFF000ull;
  while (todo) {
    int a = ctz64(todo);
    todo &= todo - 1;
    int len = contraction_len(at, win_base + a, (int64_t)0, icase);
    if (!len) continue;
    // the whole match must lie inside the document: no doc start in (a, a+len)
    uint64_t inside = ((1ull << len) - 2ull) << a;  // bits a+1 .. a+len-1
    if (w.DS & inside) continue;
    cs |= 1ull << a;
    start &= ~(1ull << (a + 1));
    if (a + len < 64) start |= 1ull << (a + len);
  }
  *contr_start_out = cs;
  return start;
}

// ---------------------------------------------------------------------------------------------- GPT-2
// byte_level.rs:44   's|'t|'re|'ve|'m|'ll|'d| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+
template <class ByteAt>
B2T_HD BoundaryOut boundaries_gpt2(const Window& w, int64_t win_base, const ByteAt& at) {
  const uint64_t nDS = ~w.DS;
  const uint64_t O = ~(w.L | w.N | w.S);
  const uint64_t pL = (w.L << 1) & nDS, pN = (w.N << 1) & nDS, pO = (O << 1) & nDS, pS = (w.S << 1) & nDS,
                 pSP = (w.SP << 1) & nDS;
  // non-whitespace char: starts a match unless same class as the previous char or the previous char is U+0020
  uint64_t same = (w.L & pL) | (w.N & pN) | (O & pO);
  uint64_t start = w.lead & ~w.S & ~same & ~pSP;
  // whitespace char: run start, or last char of a run that is followed by a non-space (\s+(?!\S) gives it back)
  uint64_t lastbyte_next_nonS = w.S & (~w.S >> 1) & (nDS >> 1);
  uint64_t lastchar = last_byte_flag_to_lead(lastbyte_next_nonS, w.lead) & w.S;
  start |= w.lead & w.S & (~pS | lastchar);
  start |= w.DS;
  // contractions: the apostrophe must sit at a match start => previous char is L, N, non-U+0020 whitespace, or none
  uint64_t cand = w.AP & (pL | pN | (pS & ~pSP) | w.DS);
  uint64_t cs;
  if (cand) start = apply_contractions(start, cand, w, win_base, at, false, &cs);
  BoundaryOut o;
  o.start = (uint32_t)((start & w.lead) >> 16);
  o.drop = 0;
  o.slow = 0;
  return o;
}

// ---------------------------------------------------------------------------------------------- Llama-3 / tiktoken
// (?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+
//
// n_phase_in: number of \p{N} characters (mod 3) of the digit run that continues into window bit 16 from before
// the window; only consulted when the run really starts before window bit 0 (see `slow`).
// zone_in / tail_in: run properties arriving from outside the window (only consulted by the slow-path caller).
struct LlamaCarry {
  int n_count_before_window;  // \p{N} chars of the current run before window bit 0 (if the run covers bit 0)
  bool zone_before_window;    // byte just before window bit 0 is in the leading-newline zone
  bool tail_after_window;     // byte just after window bit 63 is in the newline-free tail
};

template <class ByteAt>
B2T_HD BoundaryOut boundaries_llama3(const Window& w, int64_t win_base, const ByteAt& at, const LlamaCarry& carry) {
  const uint64_t nDS = ~w.DS;
  const uint64_t O = ~(w.L | w.N | w.S);
  const uint64_t pL = (w.L << 1) & nDS, pO = (O << 1) & nDS, pS = (w.S << 1) & nDS, pSP = (w.SP << 1) & nDS,
                 pNL = (w.NL << 1) & nDS;
  uint32_t slow = 0;

  // O char at a match start: previous char is neither O nor U+0020
  uint64_t ms_O = w.lead & O & ~(pO | pSP);
  // contractions first (they change which letter starts a match)
  uint64_t cand = w.AP & ms_O;
  uint64_t forced = 0, contr = 0;
  if (cand) {
    uint64_t s0 = 0;
    uint64_t s1 = apply_contractions(s0, cand, w, win_base, at, true, &contr);
    forced = s1;  // bits set = forced starts right after a contraction
  }

  // ---- letters:  [^\r\n\p{L}\p{N}]?\p{L}+
  uint64_t startL = w.lead & w.L & ~pL;
  uint64_t absorbO = to_next_lead(ms_O & ~contr, w.lead) & nDS;  // previous char is an O at a match start (not a contraction)
  uint64_t absorbS = pS & ~pNL;                                  // previous char is non-newline whitespace (always a match start)
  uint64_t start = startL & ~absorbO & ~absorbS;
  start &= ~(contr << 1);  // the letter right after a contraction apostrophe is inside the contraction
  start |= forced;

  // ---- other:  ?[^\s\p{L}\p{N}]+[\r\n]*
  start |= w.lead & O & ~pO & ~pSP;

  // ---- digits: \p{N}{1,3}: run start, then every third character
  uint64_t Nlead = w.N & w.lead;
  if (Nlead & OWN) {
    // window bit 0 has no visible predecessor: treat it as continuing, the carry says how many came before
    uint64_t runstart = Nlead & (w.DS | ~((w.N << 1) | 1ull));
    // phase of the first N lead in own region
    uint64_t own_n = Nlead & OWN;
    int cnt = 0;
    int first = ctz64(own_n);
    if (!((runstart >> first) & 1ull)) {
      // the run started earlier: find its start inside the window
      uint64_t below = runstart & ((1ull << first) - 1ull);
      if (below) {
        int rs = 63 - clz64(below);
        cnt = popc64(Nlead & ((1ull << first) - 1ull) & ~((1ull << rs) - 1ull));
      } else {
        // run covers window bit 0: need the count from before the window
        cnt = carry.n_count_before_window + popc64(Nlead & ((1ull << first) - 1ull));
        slow |= 1u;
      }
    }
    uint64_t todo = own_n;
    while (todo) {
      int p = ctz64(todo);
      todo &= todo - 1;
      if ((runstart >> p) & 1ull) cnt = 0;
      if (cnt % 3 == 0) start |= 1ull << p;
      ++cnt;
    }
  }

  // ---- whitespace
  if (w.S) {
    uint64_t startS = w.lead & w.S;
    // leading-newline zone: newlines right after an O run are swallowed by its [\r\n]*
    uint64_t zone_seed = w.NL & pO;
    if (carry.zone_before_window) zone_seed |= w.NL & 1ull & nDS;
    uint64_t zone = prop_fwd(zone_seed, w.NL & nDS);
    // newline-free tail: non-newline whitespace from here to the end of the run
    uint64_t R2 = w.S & ~w.NL;
    uint64_t tail_seed = R2 & ((~w.S >> 1) | (w.DS >> 1));
    if (carry.tail_after_window) tail_seed |= R2 & (1ull << 63);
    uint64_t tail = prop_bwd(tail_seed, R2 & (nDS >> 1));
    // does any run that matters reach a window edge?
    // (the zone of window bit 15 decides own bit 16 through Ba, hence OWN | bit 15)
    if ((w.NL & 1ull) && (prop_fwd(w.NL & 1ull, w.NL & nDS) & (OWN | 0x8000ull))) slow |= 1u;
    if ((R2 >> 63) && (prop_bwd(R2 & (1ull << 63), R2 & (nDS >> 1)) & OWN)) slow |= 1u;

    uint64_t B1 = startS & ~pS & ~zone;                      // first char of the run (unless swallowed)
    uint64_t Ba = startS & pS & ~zone & (zone << 1);         // first char after the swallowed newlines
    uint64_t Bb = startS & pNL & tail;                       // char after the last newline of the run
    uint64_t lastbyte_next_nonS = w.S & (~w.S >> 1) & (nDS >> 1);
    uint64_t lastchar = last_byte_flag_to_lead(lastbyte_next_nonS, w.lead) & w.S;
    uint64_t Bc = lastchar & ~w.NL & ((R2 << 1) & nDS);      // \s+(?!\S) gives the last char back
    start |= B1 | Ba | Bb | Bc;
  }
  start |= w.DS;
  BoundaryOut o;
  o.start = (uint32_t)((start & w.lead) >> 16);
  o.drop = 0;
  o.slow = slow;
  return o;
}

// ---------------------------------------------------------------------------------------------- Whitespace
// whitespace.rs:22  \w+|[^\w\s]+ ; the whitespace in between is removed.  Classes: L slot = \w, S = \s.
B2T_HD BoundaryOut boundaries_whitespace(const Window& w) {
  const uint64_t nDS = ~w.DS;
  const uint64_t P = ~(w.L | w.S);
  const uint64_t pW = (w.L << 1) & nDS, pS = (w.S << 1) & nDS, pP = (P << 1) & nDS;
  uint64_t same = (w.L & pW) | (w.S & pS) | (P & pP);
  uint64_t start = (w.lead & ~same) | w.DS;
  BoundaryOut o;
  o.start = (uint32_t)((start & w.lead) >> 16);
  o.drop = (uint32_t)((start & w.lead & w.S) >> 16);
  o.slow = 0;
  return o;
}

}  // namespace b2t

// ---------------------------------------------------------------------------------------------- slow path (Llama-3)
// Run properties arriving from outside the 64-byte window of `chunk`.  masks(k) / ds(k) give the class masks and the
// doc-start word of any chunk k in [0, n_chunks).  Steps are chunk-wise (32 bytes per iteration).
namespace b2t {
#if defined(__CUDA_ARCH__)
B2T_HD int clz32(uint32_t x) { return __clz((int)x); }
#else
B2T_HD int clz32(uint32_t x) { return x ? __builtin_clz(x) : 32; }
#endif
B2T_HD uint32_t bits_below(int n) { return n >= 32 ? 0xFFFFFFFFu : ((1u << n) - 1u); }

template <class MaskAt, class DsAt>
B2T_HD LlamaCarry llama_carry(int64_t chunk, int64_t n_chunks, const MaskAt& masks, const DsAt& ds) {
  LlamaCarry c;
  c.n_count_before_window = 0;
  c.zone_before_window = false;
  c.tail_after_window = false;
  // (1) \p{N} characters of the run that ends right before the window (window bit 0 = byte 16 of chunk-1)
  {
    int64_t k = chunk - 1;
    int hi = 16, cnt = 0;
    while (k >= 0) {
      ChunkMasks M = masks(k);
      uint32_t d = ds(k), lo_mask = bits_below(hi);
      uint32_t non = ~M.N & lo_mask;
      int runlow = non ? 32 - clz32(non) : 0;
      uint32_t run = lo_mask & ~bits_below(runlow);
      uint32_t dsin = d & run;
      if (dsin) { run &= ~bits_below(31 - clz32(dsin)); cnt += popc32(M.N & M.lead & run); break; }
      cnt += popc32(M.N & M.lead & run);
      if (runlow > 0 || run == 0u) break;
      --k; hi = 32;
    }
    c.n_count_before_window = cnt;
  }
  // (2) is the byte before the window an O char, or a newline inside a leading-newline zone?
  {
    int64_t k = chunk - 1;
    int hi = 16;
    bool res = false;
    while (k >= 0) {
      ChunkMasks M = masks(k);
      uint32_t d = ds(k), lo_mask = bits_below(hi);
      uint32_t non = ~M.NL & lo_mask;
      int runlow = non ? 32 - clz32(non) : 0;
      uint32_t run = lo_mask & ~bits_below(runlow);
      if (d & run) { res = false; break; }
      if (runlow > 0) { uint32_t O = ~(M.L | M.N | M.S); res = (O >> (runlow - 1)) & 1u; break; }
      if (k == 0) { res = false; break; }
      --k; hi = 32;
    }
    c.zone_before_window = res;
  }
  // (3) does the non-newline whitespace continue newline-free to the end of its run after the window?
  {
    int64_t k = chunk + 1;
    int lo = 16;
    bool res = true;
    while (true) {
      if (k >= n_chunks) { res = true; break; }
      ChunkMasks M = masks(k);
      uint32_t d = ds(k);
      uint32_t stop = (d | ~(M.S & ~M.NL)) & ~bits_below(lo);
      if (stop) {
        int s = ctz32(stop);
        res = ((d >> s) & 1u) ? true : !((M.S >> s) & 1u);
        break;
      }
      ++k; lo = 0;
    }
    c.tail_after_window = res;
  }
  return c;
}
}  // namespace b2t
