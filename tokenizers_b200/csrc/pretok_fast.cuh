// pretok_fast.cuh -- bit-sliced classification and 32-bit boundary algebra of the pre-tokenization scan (host + device).
//
// This is the fast path of K1 (pretok_stream_kernel in pretok_kernels.cuh).  It computes exactly what the window code of
// pretok_logic.cuh computes -- the split points of
//   pre_tokenizers/byte_level.rs:43-46,119-131 (GPT-2 pattern), pre_tokenizers/whitespace.rs:20-29 (\w+|[^\w\s]+)
// -- with about a third of the instructions, because the kernel is bound by the integer pipe, not by HBM:
//   1. the 32 bytes of a chunk are transposed into 8 bit planes (bitslice32: 16 byte permutes + 12 register-pair
//      exchanges), after which every class test is boolean logic on 32 positions at once;
//   2. non-ASCII characters of the blocks that dominate real text (Latin-1/Extended, Greek, Cyrillic, CJK, Hangul,
//      emoji, general punctuation) are classified by boolean functions of their first two or three bytes
//      (`certain_*`, checked against the full class table for every code point by tests/test_pretok_fast_cpu.py);
//      the rest take a table look-up per character (resolve_uncertain);
//   3. the boundary predicates work on the chunk's own 32-bit masks, the neighbours contribute single bits
//      (funnel shifts) instead of 64-bit windows.
// The window code stays as the exact fallback for the one case the fast algebra does not cover (a multi-byte
// whitespace character that straddles the chunk end) and as the Llama-3 algebra.
// Everything here is pure so that tests/native/pretok_emul.cpp runs exactly this code on the CPU.
#pragma once
#include "pretok_logic.cuh"

namespace b2t {

// ---------------------------------------------------------------------------------------------- primitives
#if defined(__CUDA_ARCH__)
B2T_HD uint32_t bperm(uint32_t x, uint32_t y, uint32_t s) { return __byte_perm(x, y, s); }
B2T_HD uint32_t fsl(uint32_t lo, uint32_t hi, int k) { return __funnelshift_l(lo, hi, k); }   // (hi:lo << k) >> 32
B2T_HD uint32_t fsr(uint32_t lo, uint32_t hi, int k) { return __funnelshift_r(lo, hi, k); }   // (hi:lo >> k) & 0xFFFFFFFF
#else
B2T_HD uint32_t bperm(uint32_t x, uint32_t y, uint32_t s) {
  uint64_t v = ((uint64_t)y << 32) | x;
  uint32_t r = 0;
  for (int i = 0; i < 4; ++i) r |= (uint32_t)((v >> (8 * ((s >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
  return r;
}
B2T_HD uint32_t fsl(uint32_t lo, uint32_t hi, int k) { return (uint32_t)(((((uint64_t)hi << 32) | lo) << k) >> 32); }
B2T_HD uint32_t fsr(uint32_t lo, uint32_t hi, int k) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> k); }
#endif
// x >> K for a constant K.  On the device as a multiply-high: the shift units share the integer pipe with the logic
// ops that bound this kernel, the multiplier sits on the other pipe (kept switchable, off by default).
#ifndef B2T_SHR_MULHI
#define B2T_SHR_MULHI 0
#endif
template <int K>
B2T_HD uint32_t shr(uint32_t x) {
#if defined(__CUDA_ARCH__) && B2T_SHR_MULHI
  return __umulhi(x, 1u << (32 - K));
#else
  return x >> K;
#endif
}
// 3-input look-up: bit (a b c) of TB.  Written as a sum of minterms over three variables, which nvcc folds into ONE LOP3.
// (An inline-asm lop3 here once produced wrong class masks when the call sat next to a warp vote -- seen on the GPU
// against the CPU run of this very file -- so the compiler does the folding.)
template <uint32_t TB>
B2T_HD uint32_t lop3(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if ((TB >> i) & 1u) d |= ((i & 4) ? a : ~a) & ((i & 2) ? b : ~b) & ((i & 1) ? c : ~c);
  return d;
}

// Boolean function of NV variables x[0..NV-1] given by its truth table T (bit i = value at x = i), evaluated on 32
// positions at once: a tree of 3-input look-ups (one LOP3 each) and 2:1 selects, pruned at compile time.
template <uint64_t T, int NV>
B2T_HD uint32_t tt_eval(const uint32_t* x) {
  if constexpr (NV == 3) {
    constexpr uint32_t tb = (uint32_t)(T & 0xFFu);
    if constexpr (tb == 0u) return 0u;
    else if constexpr (tb == 0xFFu) return ~0u;
    else return lop3<tb>(x[2], x[1], x[0]);
  } else {
    constexpr int half = 1 << (NV - 1);
    constexpr uint64_t mask = (1ull << half) - 1ull;
    constexpr uint64_t lo = T & mask, hi = (T >> half) & mask;
    if constexpr (lo == hi) return tt_eval<lo, NV - 1>(x);
    else {
      const uint32_t a = tt_eval<lo, NV - 1>(x), b = tt_eval<hi, NV - 1>(x);
      return (x[NV - 1] & b) | (~x[NV - 1] & a);
    }
  }
}

// ---------------------------------------------------------------------------------------------- bit slicing
// w[0..7]: the chunk's 32 bytes as little-endian words.  b[j] bit p = bit j of byte p.
// The three exchange masks are passed at RUN TIME (kernel parameters): with a compile-time mask nvcc splits
// (x & M) | (y & ~M) into two look-ups with two immediates; with M in a register / constant bank it is one LOP3.
struct SwapMasks { uint32_t m1, m2, m4; };   // 0x55555555, 0x33333333, 0x0F0F0F0F
template <uint32_t D>
B2T_HD void plane_swap(uint32_t& a, uint32_t& b, uint32_t M) {
  const uint32_t na = (a & M) | ((b << D) & ~M);
  const uint32_t nb = (shr<D>(a) & M) | (b & ~M);
  a = na; b = nb;
}
B2T_HD void bitslice32(const uint32_t w[8], uint32_t b[8], SwapMasks k = SwapMasks{0x55555555u, 0x33333333u, 0x0F0F0F0Fu}) {
  // byte permutation: b[k] <- [byte k, byte k+8, byte k+16, byte k+24]
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t t0 = bperm(w[h], w[h + 2], 0x5140u), t1 = bperm(w[h + 4], w[h + 6], 0x5140u);
    const uint32_t t2 = bperm(w[h], w[h + 2], 0x7362u), t3 = bperm(w[h + 4], w[h + 6], 0x7362u);
    b[4 * h + 0] = bperm(t0, t1, 0x5410u); b[4 * h + 1] = bperm(t0, t1, 0x7632u);
    b[4 * h + 2] = bperm(t2, t3, 0x5410u); b[4 * h + 3] = bperm(t2, t3, 0x7632u);
  }
  // exchange register-index bit i with bit-index bit i (i = 0, 1, 2)
  plane_swap<1>(b[0], b[1], k.m1); plane_swap<1>(b[2], b[3], k.m1); plane_swap<1>(b[4], b[5], k.m1); plane_swap<1>(b[6], b[7], k.m1);
  plane_swap<2>(b[0], b[2], k.m2); plane_swap<2>(b[1], b[3], k.m2); plane_swap<2>(b[4], b[6], k.m2); plane_swap<2>(b[5], b[7], k.m2);
  plane_swap<4>(b[0], b[4], k.m4); plane_swap<4>(b[1], b[5], k.m4); plane_swap<4>(b[2], b[6], k.m4); plane_swap<4>(b[3], b[7], k.m4);
}

// ---------------------------------------------------------------------------------------------- classification
struct FastCls {
  uint32_t lead, cont, hi;        // byte starts a character / is a continuation byte / is not ASCII
  uint32_t L, N, S, SP, AP, NL;   // class masks; after fill_own + spill_in every byte carries its character's class
  uint32_t A2, A3;                // GPT-2: apostrophes followed by s|t|m|d / by re|ve|ll inside the chunk (AP keeps only the
                                  // apostrophes whose letters lie past the chunk end: they take the per-apostrophe path)
  uint32_t unc;                   // non-ASCII lead bytes whose class still needs the table (resolve_uncertain)
};

// Lead bytes (index = byte & 63) whose whole subtree has one class in BOTH class schemes (onig \p{L}.. and rust \w..):
// C4-CA D0 D1 D3 DA E5-E9 EB EC are letters, EE F1 F2 F4 are "other".  Verified by tests/test_pretok_fast_cpu.py.
constexpr uint64_t LEAD_ALL_L = 0x1BE0040B07F0ull;
constexpr uint64_t LEAD_ALL_O = 0x16400000000000ull;

template <int KIND>
B2T_HD FastCls classify_planes(const uint32_t b[8], uint32_t valid) {
  const uint32_t b0 = b[0], b1 = b[1], b2 = b[2], b3 = b[3], b4 = b[4], b5 = b[5], b6 = b[6], b7 = b[7];
  FastCls m;
  m.hi = b7;
  m.cont = b7 & ~b6;
  m.lead = ~m.cont & valid;
  // ---- ASCII
  const uint32_t lo3 = b2 | (b1 & b0);                       // low 3 bits >= 3
  const uint32_t alpha = ~b7 & b6 & (b4 | b3 | b2 | b1 | b0) & ~(b4 & b3 & lo3);   // low 5 bits in 1..26
  const uint32_t c30 = ~b7 & ~b6 & b5 & b4;                  // 0x30..0x3F
  const uint32_t digit = c30 & ~(b3 & (b2 | b1));            // 0x30..0x39
  const uint32_t c20 = ~b7 & ~b6 & b5 & ~b4;                 // 0x20..0x2F
  const uint32_t sp = c20 & ~(b3 | b2 | b1 | b0);            // 0x20
  const uint32_t c00 = ~(b7 | b6 | b5 | b4);                 // 0x00..0x0F
  const uint32_t wsctl = c00 & b3 & (b2 | b1 | b0) & ~(b2 & b1);   // 0x09..0x0D
  m.SP = sp;
  m.S = sp | wsctl;
  m.A2 = 0u; m.A3 = 0u;
  if (KIND == PT_WHITESPACE) {
    m.L = alpha | digit | (~b7 & b6 & ~b5 & b4 & b3 & b2 & b1 & b0);   // \w on ASCII: letters, digits, '_' (0x5F)
    m.N = 0u; m.AP = 0u; m.NL = 0u;
  } else if (KIND == PT_BERT) {
    // BertPreTokenizer on ASCII: whitespace as above, punctuation = is_ascii_punctuation, words = everything else, i.e.
    // letters, digits, the control characters that are not whitespace, DEL
    const uint32_t ctl = ~(b7 | b6 | b5) & ~wsctl;                      // 0x00..0x1F without 0x09..0x0D
    m.L = alpha | digit | ctl | (~b7 & b6 & b5 & b4 & b3 & b2 & b1 & b0);
    m.N = 0u; m.AP = 0u; m.NL = 0u;
  } else {
    m.L = alpha; m.N = digit;
    m.AP = c20 & ~b3 & b2 & b1 & b0;                         // 0x27
    if (KIND == PT_GPT2) {
      // 's 't 'm 'd / 're 've 'll (case-sensitive): letter tests on the low 5 bits of 0x60..0x7F
      const uint32_t lower = ~b7 & b6 & b5;
      const uint32_t x5[5] = {b0, b1, b2, b3, b4};
      const uint32_t stmd = lower & tt_eval<(1ull << 19) | (1ull << 20) | (1ull << 13) | (1ull << 4), 5>(x5);
      const uint32_t rv = lower & tt_eval<(1ull << 18) | (1ull << 22), 5>(x5);
      const uint32_t le = lower & tt_eval<(1ull << 5), 5>(x5), ll = lower & tt_eval<(1ull << 12), 5>(x5);
      const uint32_t f3 = (rv & shr<1>(le)) | (ll & shr<1>(ll));    // first letter of re / ve / ll (both letters inside the chunk)
      m.A2 = m.AP & shr<1>(stmd);
      m.A3 = m.AP & shr<1>(f3);
      // undecidable here: the apostrophe at bit 31, and the one at bit 30 when its letter is r / v / l
      m.AP &= 0x80000000u | (0x40000000u & shr<1>(rv | ll));
    }
    m.NL = KIND == PT_LLAMA3 ? (c00 & b3 & ~(b2 ^ b0) & (b1 ^ b0)) : 0u;   // 0x0A, 0x0D
  }
  // ---- non-ASCII: characters whose class follows from their first bytes
  m.unc = 0u;
  if (KIND == PT_BERT) {
    m.unc = b7 & b6 & valid;   // no shortcuts for BERT's classes: every non-ASCII character takes the table
  } else if (b7) {
    const uint32_t nlead = b7 & b6 & valid;                  // non-ASCII lead bytes
    // conditions on a continuation byte (its low 6 bits), moved to the position of the byte before it; a lead byte at
    // position 31 sees zeros and stays uncertain
    const uint32_t x54 = b5 & b4, o54 = b5 | b4;
    const uint32_t k_c3 = shr<1>(~(b4 & ~b3 & b2 & b1 & b0));            // != 0x97, 0xB7     (U+00D7, U+00F7)
    const uint32_t k_ce = shr<1>(b5 & (b4 | b3 | lo3));                  // >= 0xA3           (U+03A3..)
    const uint32_t k_cf = shr<1>(~(x54 & ~b3 & b2 & b1 & ~b0));          // != 0xB6           (U+03F6)
    const uint32_t k_e4 = shr<1>(~(x54 & ~b3 & b2 & b1 & b0));           // != 0xB7           (U+4DC0..U+4DFF)
    const uint32_t k_e3 = shr<1>(o54);                                   // >= 0x90           (U+3400..)
    const uint32_t k_ea = shr<1>(x54);                                   // >= 0xB0           (U+AC00..)
    const uint32_t k_ed = shr<1>(~b5 & ~(b4 & b3 & b2 & b1));            // <= 0x9D           (..U+D77F)
    const uint32_t z6 = ~(b5 | b4 | b3 | b2 | b1 | b0);                  // == 0x80
    const uint32_t z6s = shr<1>(z6);
    const uint32_t k_e2 = z6s & shr<2>((~b5 & b4) | (b5 & ~b4 & ~b3));   // E2 80 90..A7      (U+2010..U+2027)
    const uint32_t f9f = ~b5 & b4 & b3 & b2 & b1 & b0;                   // == 0x9F
    const uint32_t k_f0 = shr<1>(f9f) & shr<2>(~((~(b5 | b4 | b3) & b2) | (b5 & ~b4 & b3 & b2 & b1 & b0)));  // F0 9F, third byte not 84..87, AF
    const uint32_t x[6] = {b0, b1, b2, b3, b4, b5};
    // lead byte & 63 = 8 * row + col: one look-up per row (b5 b4 b3) and per column (b2 b1 b0) that a rule names
    const uint32_t r0 = lop3<0x01>(b5, b4, b3), r1 = lop3<0x02>(b5, b4, b3), r4 = lop3<0x10>(b5, b4, b3),
                   r5 = lop3<0x20>(b5, b4, b3), r6 = lop3<0x40>(b5, b4, b3);
    const uint32_t c0 = lop3<0x01>(b2, b1, b0), c2 = lop3<0x04>(b2, b1, b0), c3 = lop3<0x08>(b2, b1, b0),
                   c4 = lop3<0x10>(b2, b1, b0), c5 = lop3<0x20>(b2, b1, b0);
    const uint32_t row0 = c3 & k_c3;                                        // C3
    const uint32_t row1 = b2 & b1 & ((b0 & k_cf) | (~b0 & k_ce));           // CE, CF
    const uint32_t row4 = (c3 & k_e3) | (c4 & k_e4);                        // E3, E4
    const uint32_t row5 = (c2 & k_ea) | (c5 & k_ed);                        // EA, ED
    uint32_t cl = tt_eval<LEAD_ALL_L, 6>(x) | (r0 & row0) | (r1 & row1) | (r4 & row4) | (r5 & row5);
    uint32_t co = tt_eval<LEAD_ALL_O, 6>(x) | (r4 & c2 & k_e2) | (r6 & c0 & k_f0);   // E2, F0
    // the two multi-byte spaces of everyday text: U+00A0 (C2 A0) and U+3000 (E3 80 80)
    uint32_t cs = (r0 & c2 & shr<1>(b5 & ~(b4 | b3 | b2 | b1 | b0))) | (r4 & c3 & z6s & shr<2>(z6));
    cl &= nlead; co &= nlead; cs &= nlead;
    m.L |= cl; m.S |= cs;
    m.unc = nlead & ~(cl | co | cs);
  }
  return m;
}

// Table look-up for the characters classify_planes left open (one per set bit of m.unc).  at4(q) = the four bytes at
// q..q+3 as a little-endian word (bytes past the end of the character are ignored; the text is valid UTF-8).
template <class At4, class Pos>
B2T_HD void resolve_uncertain(FastCls& m, const At4& at4, Pos base, const uint32_t* __restrict__ cls_tbl) {
  uint32_t todo = m.unc;
  while (todo) {
    const int p = ctz32(todo);
    todo &= todo - 1u;
    const uint32_t v = at4(base + (Pos)p);
    const uint32_t b0 = v & 0xFFu;
    const int len = 2 + (b0 >= 0xE0u) + (b0 >= 0xF0u);
    // branch-free decode: the low 6 bits of all four bytes as if the character had 4 bytes, shifted down by the bytes
    // it does not have, lead-byte marker bits masked off
    const uint32_t t24 = ((v & 0x3Fu) << 18) | ((v << 4) & 0x3F000u) | ((v >> 10) & 0xFC0u) | ((v >> 24) & 0x3Fu);
    uint32_t cp = (t24 >> (6 * (4 - len))) & ((2u << (5 * len)) - 1u);
    cp = cp < 0x110000u ? cp : 0x10FFFFu;
    const uint32_t c = class_of(cls_tbl, cp);
    const uint32_t bit = 1u << p;
    m.L |= c == CLS_L ? bit : 0u; m.N |= c == CLS_N ? bit : 0u; m.S |= c == CLS_S ? bit : 0u;
  }
  m.unc = 0u;
}

// Continuation bytes inherit the class of their lead byte (inside the chunk).
B2T_HD void fill_own(FastCls& m) {
  const uint32_t c1 = m.cont, c2 = m.cont & (m.cont << 1);
  uint32_t x;
  x = m.L; x |= (x << 1) & c1; x |= (x << 2) & c2; m.L = x;
  x = m.N; x |= (x << 1) & c1; x |= (x << 2) & c2; m.N = x;
  x = m.S; x |= (x << 1) & c1; x |= (x << 2) & c2; m.S = x;
}
// ... and of the character that started in the previous chunk (pL/pN/pS: bit 31 = class of that chunk's last byte).
B2T_HD void spill_in(FastCls& m, uint32_t pL, uint32_t pN, uint32_t pS) {
  const uint32_t low = m.cont & ~(m.cont + 1u);   // the continuation bytes the chunk starts with
  m.L |= low & (0u - (pL >> 31));
  m.N |= low & (0u - (pN >> 31));
  m.S |= low & (0u - (pS >> 31));
}

// What a chunk needs from the one before it: bit 31 of these words = class of the previous chunk's last byte.
struct PrevTop { uint32_t L, N, S, SP; };
// What a chunk hands to the next one when a contraction reaches across the chunk end (bits 0..2: forced starts,
// bit 8: position 0 of the next chunk is the letter right after the apostrophe and must not start a split).
struct Overflow { uint32_t bits; };

struct FastOut {
  uint32_t start, drop;
  uint32_t fallback;   // 1: the chunk needs the exact window code (a multi-byte whitespace character straddles its end)
  Overflow ov;         // to be applied to the NEXT chunk with apply_overflow
};

B2T_HD uint32_t apply_overflow(uint32_t start, uint32_t lead, Overflow in) {
  return ((start & ~(in.bits >> 8)) | (in.bits & 7u)) & lead;
}

// byte_level.rs:44   's|'t|'re|'ve|'m|'ll|'d| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+
// next_lead0 / next_S0: bit 0 of the next chunk's lead / S masks; ds / ds_next: doc-start words of this and the next chunk.
// The result does not contain the previous chunk's overflow yet (apply_overflow).
// Contraction length for the apostrophe whose following two bytes are b1, b2 (GPT-2: case-sensitive): 0 / 2 / 3.
B2T_HD int contraction_len2(uint32_t a, uint32_t b) {
  if (a == 's' || a == 't' || a == 'm' || a == 'd') return 2;
  if ((a == 'r' || a == 'v') && b == 'e') return 3;
  if (a == 'l' && b == 'l') return 3;
  return 0;
}

// The bit the whitespace rule leaves open in fast_gpt2 when it is called with next_lead0 = next_S0 = 1: whether the
// whitespace character that ends the chunk (or straddles its end) is the last one of its run and followed by a
// non-space of the same document -- then \s+(?!\S) gives it back and it starts a split of its own.
//   s31: bit 31 of the chunk's S mask; lead: its lead mask; nlead / nS: bits 0..3 of the NEXT chunk's lead / S masks
//   (after fill and spill-in); ds_next: the next chunk's doc-start word.
B2T_HD uint32_t finalize_gpt2(uint32_t start, uint32_t lead, uint32_t s31, uint32_t nlead, uint32_t nS, uint32_t ds_next) {
  if (s31) {
    const int k = ctz32((nlead & 7u) | 8u);   // bytes of my last character that lie in the next chunk (3: nothing follows)
    if (k < 3 && lead && !((nS >> k) & 1u) && !((ds_next >> k) & 1u)) start |= 0x80000000u >> clz32(lead);
  }
  return start;
}

template <class At4, class Pos>
B2T_HD FastOut fast_gpt2(const FastCls& m, const PrevTop& p, uint32_t next_lead0, uint32_t next_S0, uint32_t ds, uint32_t ds_next,
                         Pos base, const At4& at4) {
  FastOut o;
  o.drop = 0u; o.fallback = 0u; o.ov.bits = 0u;
  const uint32_t O = ~(m.L | m.N | m.S);
  const uint32_t pL = fsl(p.L, m.L, 1), pN = fsl(p.N, m.N, 1), pS = fsl(p.S, m.S, 1), pSP = fsl(p.SP, m.SP, 1);
  const uint32_t pO = ~(pL | pN | pS);
  const uint32_t same = (m.L & pL) | (m.N & pN) | (O & pO);
  uint32_t start = ~m.S & ~same & ~pSP;
  // whitespace: run start, or last character of a run that is followed by a non-space of the same document
  const uint32_t nS0 = next_lead0 ? next_S0 : (m.S >> 31);        // class of the byte after the chunk
  const uint32_t nS = (m.S >> 1) | (nS0 << 31);
  const uint32_t nDS = fsr(ds, ds_next, 1);
  const uint32_t E = m.S & ~nS & ~nDS;                             // last byte of such a run
  uint32_t lastchar = E;
  if (E & m.cont) {                                                // rare: the run ends with a multi-byte space
    const uint32_t e1 = (E & m.cont) >> 1, e2 = (e1 & m.cont) >> 1;
    lastchar = E | e1 | e2;
  }
  if (((m.S & m.hi) >> 31) & (next_lead0 ^ 1u)) o.fallback = 1u;  // its bytes continue in the next chunk
  start |= m.S & (~pS | lastchar);
  start |= ds;
  // contractions: the apostrophe must sit at a match start, the whole match inside the document
  const uint32_t at_start = pL | pN | (pS & ~pSP) | ds;
  {
    const uint32_t nDS2 = fsr(ds, ds_next, 2);
    const uint32_t c2 = m.A2 & at_start & ~nDS, c3 = m.A3 & at_start & ~nDS & ~nDS2, cc = c2 | c3;
    start = (start & ~(cc << 1)) | (c2 << 2) | (c3 << 3);       // the letter after the apostrophe does not start a split, the character after the match does
    o.ov.bits = ((c2 >> 30) | (c3 >> 29)) & 1u;                  // 's at bit 30 / 're at bit 29: that character is the next chunk's first
  }
  uint32_t cand = m.AP & at_start;                                // letters in the next chunk: one at a time, from the bytes
  if (cand) {
    const uint64_t ds64 = (uint64_t)ds | ((uint64_t)ds_next << 32);
    uint64_t set = 0, clr = 0;
    while (cand) {
      const int a = ctz32(cand);
      cand &= cand - 1u;
      const uint32_t v = at4(base + (Pos)a);
      const int len = contraction_len2((v >> 8) & 0xFFu, (v >> 16) & 0xFFu);
      if (!len) continue;
      if (ds64 & (((1ull << len) - 2ull) << a)) continue;          // the match must lie inside the document
      clr |= 1ull << (a + 1);
      set |= 1ull << (a + len);
    }
    start = (start & ~(uint32_t)clr) | (uint32_t)set;
    o.ov.bits |= (uint32_t)(set >> 32) | ((uint32_t)(clr >> 32) << 8);
  }
  o.start = start & m.lead;
  return o;
}

// pre_tokenizers/bert.rs:14-18: split on whitespace (removed), then every punctuation character on its own (Isolated).
// L slot = word characters, S = whitespace, everything else is punctuation and never joins its neighbour.
B2T_HD FastOut fast_bert(const FastCls& m, const PrevTop& p, uint32_t ds) {
  FastOut o;
  o.fallback = 0u; o.ov.bits = 0u;
  const uint32_t pW = fsl(p.L, m.L, 1), pS = fsl(p.S, m.S, 1);
  const uint32_t same = (m.L & pW) | (m.S & pS);
  const uint32_t start = (~same | ds) & m.lead;
  o.start = start;
  o.drop = start & m.S;
  return o;
}

// whitespace.rs:22  \w+|[^\w\s]+ ; the whitespace in between is removed.  L slot = \w, S = \s.
B2T_HD FastOut fast_whitespace(const FastCls& m, const PrevTop& p, uint32_t ds) {
  FastOut o;
  o.fallback = 0u; o.ov.bits = 0u;
  const uint32_t P = ~(m.L | m.S);
  const uint32_t pW = fsl(p.L, m.L, 1), pS = fsl(p.S, m.S, 1);
  const uint32_t pP = ~(pW | pS);
  const uint32_t same = (m.L & pW) | (m.S & pS) | (P & pP);
  const uint32_t start = (~same | ds) & m.lead;
  o.start = start;
  o.drop = start & m.S;
  return o;
}

}  // namespace b2t
