// host_tables.cu -- see host_tables.h
#include "host_tables.h"

#include "../../include/b2t.h"

#include <string.h>
#include <vector_types.h>

#include <algorithm>

#include "pretok_logic.cuh"
#include "unicode_ranges.inc"
#include "bert_tables.inc"

namespace b2t {

void unicode_class_table(int scheme, uint8_t* out) {
  memset(out, 0, 0x110000);
  auto fill = [&](const uint32_t (*r)[2], uint32_t cnt, uint8_t v) {
    for (uint32_t i = 0; i < cnt; ++i)
      for (uint32_t c = r[i][0]; c <= r[i][1]; ++c) out[c] = v;
  };
  if (scheme == 0) {
    fill(B2T_ONIG_L, B2T_ONIG_L_COUNT, CLS_L);
    fill(B2T_ONIG_N, B2T_ONIG_N_COUNT, CLS_N);
    fill(B2T_ONIG_S, B2T_ONIG_S_COUNT, CLS_S);
  } else if (scheme == 2) {
    // BertPreTokenizer (pre_tokenizers/bert.rs:5-19): whitespace is removed, punctuation isolated, the rest forms words
    memset(out, CLS_L, 0x110000);
    fill(B2T_BERT_PUNCT, B2T_BERT_PUNCT_COUNT, CLS_O);
    fill(B2T_BERT_WS, B2T_BERT_WS_COUNT, CLS_S);
  } else {
    fill(B2T_RUST_W, B2T_RUST_W_COUNT, CLS_L);
    fill(B2T_RUST_S, B2T_RUST_S_COUNT, CLS_S);
  }
}

void space_counts(const uint8_t* s, uint32_t len, const uint8_t* cls, uint32_t* chars, uint32_t* lead, uint32_t* trail) {
  std::vector<bool> sp;
  for (uint32_t i = 0; i < len;) {   // (a malformed sequence counts as one char per byte, not as whitespace)
    const uint8_t b = s[i];
    uint32_t n = b < 0x80 ? 1 : (b >> 5) == 6 ? 2 : (b >> 4) == 14 ? 3 : (b >> 3) == 30 ? 4 : 1;
    if (i + n > len) n = 1;
    uint32_t cp = n == 1 ? b : (uint32_t)(b & (0x7F >> n));
    for (uint32_t k = 1; k < n; ++k) cp = (cp << 6) | (s[i + k] & 63u);
    sp.push_back(cp == 0x120u || (cp < 0x110000 && cls[cp] == CLS_S && (n > 1 || b < 0x80)));
    i += n;
  }
  uint32_t l = 0, t = 0;
  while (l < sp.size() && sp[l]) ++l;
  while (t < sp.size() && sp[sp.size() - 1 - t]) ++t;
  *chars = (uint32_t)sp.size(); *lead = l; *trail = t;
}

std::vector<uint32_t> vocab_trim_counts(uint32_t n_vocab, const uint8_t* vocab_bytes, const uint32_t* vocab_off, const uint32_t* vocab_ids) {
  uint32_t n_ids = 0;
  for (uint32_t i = 0; i < n_vocab; ++i) n_ids = std::max(n_ids, vocab_ids[i] + 1);
  std::vector<uint8_t> cls(0x110000);
  unicode_class_table(1, cls.data());
  std::vector<uint32_t> out(n_ids, 0u);
  for (uint32_t i = 0; i < n_vocab; ++i) {
    uint32_t chars, lead, trail;
    space_counts(vocab_bytes + vocab_off[i], vocab_off[i + 1] - vocab_off[i], cls.data(), &chars, &lead, &trail);
    out[vocab_ids[i]] = std::min(lead, 0xFFFFu) | std::min(trail, 0xFFFFu) << 16;
  }
  return out;
}

static void utf8_append(std::string& s, uint32_t cp);

// BertNormalizer (normalizers/bert.rs:92-136) as a table: the image of every code point under the enabled steps, in the
// reference's order clean_text -> handle_chinese_chars -> strip_accents (NFD, drop Mn) -> lowercase.  Every step maps one
// character to a sequence of characters on its own; NFD's canonical reordering only moves characters with a non-zero
// combining class (817 code points decompose to one first, as the reference sees them, probed: tools/gen_bert_tables.py),
// and strip_accents drops 734 of them, so composing per character is exact for the text.  The alignment is not always:
// NormalizedString hands the original characters out in input order, so a kept mark that sorting moves takes another
// character's.  The 83 newer characters with a combining class that are NOT Mn for the reference survive: NORM_SURVIVOR,
// refused where a neighbour lets canonical ordering reach them (norm_kernels.cuh norm_survivor_refused).
void build_bert_norm(bool clean_text, bool chinese, bool strip_accents, bool lowercase, NormHost* out) {
  auto in_ranges = [](const uint32_t (*r)[2], uint32_t cnt, uint32_t c) {
    uint32_t lo = 0, hi = cnt;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (r[mid][1] < c) lo = mid + 1; else hi = mid; }
    return lo < cnt && r[lo][0] <= c;
  };
  std::unordered_map<uint32_t, std::vector<uint32_t>> nfd, low;
  for (uint32_t i = 0; i < B2T_BERT_NFD_WORDS;) { const uint32_t cp = B2T_BERT_NFD[i], k = B2T_BERT_NFD[i + 1]; nfd[cp].assign(B2T_BERT_NFD + i + 2, B2T_BERT_NFD + i + 2 + k); i += 2 + k; }
  for (uint32_t i = 0; i < B2T_BERT_LOWER_WORDS;) { const uint32_t cp = B2T_BERT_LOWER[i], k = B2T_BERT_LOWER[i + 1]; low[cp].assign(B2T_BERT_LOWER + i + 2, B2T_BERT_LOWER + i + 2 + k); i += 2 + k; }
  out->blk.assign(0x110000 >> 7, 0);
  out->ent.assign(128, 0u);            // block 0: identity everywhere
  out->pool.clear();
  out->ascii.assign(128, 0);
  std::vector<uint32_t> seq, tmp, block(128);
  std::string img;
  for (uint32_t b0 = 0; b0 < 0x110000; b0 += 128) {
    bool any = false;
    for (uint32_t c = b0; c < b0 + 128; ++c) {
      uint32_t e = NORM_IDENT;
      if (c < 0xD800 || c > 0xDFFF) {
        seq.assign(1, c);
        bool cleaned = false;     // clean_text removes it: NFD never sees it
        bool kept_mark = false;   // strip_accents keeps a piece of it with a non-zero class
        if (clean_text) {
          if (in_ranges(B2T_BERT_REMOVE, B2T_BERT_REMOVE_COUNT, c)) { seq.clear(); cleaned = true; }
          else if (in_ranges(B2T_BERT_TOSPACE, B2T_BERT_TOSPACE_COUNT, c)) seq.assign(1, 0x20u);
        }
        if (chinese && seq.size() == 1 && in_ranges(B2T_BERT_CHINESE, B2T_BERT_CHINESE_COUNT, seq[0])) { const uint32_t x = seq[0]; seq = {0x20u, x, 0x20u}; }
        if (strip_accents) {
          tmp.clear();
          for (uint32_t x : seq) {
            if (x >= 0xAC00 && x <= 0xD7A3) {   // Hangul syllable -> L V [T]
              const uint32_t si = x - 0xAC00;
              tmp.push_back(0x1100 + si / 588); tmp.push_back(0x1161 + (si % 588) / 28);
              if (si % 28) tmp.push_back(0x11A7 + si % 28);
            } else {
              auto it = nfd.find(x);
              if (it == nfd.end()) tmp.push_back(x); else tmp.insert(tmp.end(), it->second.begin(), it->second.end());
            }
          }
          seq.clear();
          for (uint32_t x : tmp)
            if (!in_ranges(B2T_BERT_MN, B2T_BERT_MN_COUNT, x)) {
              seq.push_back(x);
              kept_mark = kept_mark || in_ranges(B2T_BERT_CCC, B2T_BERT_CCC_COUNT, x);   // a kept piece with a non-zero class
            }
        }
        if (lowercase) {
          tmp.clear();
          for (uint32_t x : seq) { auto it = low.find(x); if (it == low.end()) tmp.push_back(x); else tmp.insert(tmp.end(), it->second.begin(), it->second.end()); }
          seq.swap(tmp);
        }
        // NFD starts with a non-zero combining class: canonical ordering can move it (every such character NFD keeps is a
        // NORM_SURVIVOR and every other one NORM_REMOVE, so IDENT and STRING characters start with class 0, b2t_tables.h)
        const bool reorders = strip_accents && in_ranges(B2T_BERT_CCC, B2T_BERT_CCC_COUNT, c);
        if (seq.empty()) e = NORM_REMOVE | (reorders || (strip_accents && cleaned) ? NORM_MARK_FLAG : 0u);
        else if (reorders) {
          // one of the 83 characters with a combining class that strip_accents does not drop: its image is itself, but NFD may
          // reorder it with a mark beside it -- the kernels refuse the batch when a neighbour lets it (norm_survivor_refused)
          e = (seq.size() == 1 && seq[0] == c) ? NORM_SURVIVOR : (NORM_SURVIVOR | NORM_MARK_FLAG);
        } else if (!(seq.size() == 1 && seq[0] == c)) {
          img.clear();
          for (uint32_t x : seq) utf8_append(img, x);
          const size_t src_len = c < 0x80 ? 1 : (c < 0x800 ? 2 : (c < 0x10000 ? 3 : 4));
          if (img.size() > 3 * src_len || img.size() > NORM_LEN_MASK) out->ok = false;   // (norm_write_kernel sizes its staging for 3x; holds for every character today)
          e = NORM_STRING | ((uint32_t)img.size() << 2) | ((uint32_t)out->pool.size() << 8) | (kept_mark ? NORM_TAIL_FLAG : 0u);
          out->pool.insert(out->pool.end(), img.begin(), img.end());
        }
        if (c < 128) out->ascii[c] = seq.empty() ? 0xFF : (uint8_t)seq[0];   // (an ASCII character's image is one ASCII character; 0xFF = dropped)
      }
      block[c - b0] = e;
      any = any || e != NORM_IDENT;
    }
    if (any) { out->blk[b0 >> 7] = (uint16_t)(out->ent.size() / 128); out->ent.insert(out->ent.end(), block.begin(), block.end()); }
  }
  out->pool.resize(out->pool.size() + 16, 0);
}

static void utf8_append(std::string& s, uint32_t cp) {
  if (cp < 0x80) s.push_back((char)cp);
  else if (cp < 0x800) { s.push_back((char)(0xC0 | (cp >> 6))); s.push_back((char)(0x80 | (cp & 63))); }
  else if (cp < 0x10000) { s.push_back((char)(0xE0 | (cp >> 12))); s.push_back((char)(0x80 | ((cp >> 6) & 63))); s.push_back((char)(0x80 | (cp & 63))); }
  else { s.push_back((char)(0xF0 | (cp >> 18))); s.push_back((char)(0x80 | ((cp >> 12) & 63))); s.push_back((char)(0x80 | ((cp >> 6) & 63))); s.push_back((char)(0x80 | (cp & 63))); }
}

// byte_level.rs:15-39: printable bytes keep their code point, the other 68 map to U+0100 + k in byte order
static void bytes_char_table(uint32_t cp_of_byte[256]) {
  uint32_t k = 0;
  for (int b = 0; b < 256; ++b) {
    bool printable = (b >= '!' && b <= '~') || (b >= 0xA1 && b <= 0xAC) || (b >= 0xAE && b <= 0xFF);
    cp_of_byte[b] = printable ? (uint32_t)b : 256u + k++;
  }
}

static uint32_t pow2_at_least(uint64_t x) {
  uint32_t c = 16;
  while (c < x) c <<= 1;
  return c;
}

std::string build_host_tables(int model, int pretok, int ignore_merges, uint32_t n_vocab, const uint8_t* vocab_bytes,
                              const uint32_t* vocab_off, const uint32_t* vocab_ids, uint32_t n_merges,
                              const uint8_t* merge_bytes, const uint32_t* merge_off, const char* unk_token,
                              const char* cont_prefix, uint32_t max_chars, HostTables* out, bool* vocab_err) {
  *vocab_err = false;
  // ---- class table
  {
    std::vector<uint8_t> cls(0x110000);
    unicode_class_table(pretok == PT_BERT ? 2 : (pretok == PT_WHITESPACE ? 1 : 0), cls.data());
    out->cls_packed.assign(0x110000 / 16, 0u);
    for (uint32_t c = 0; c < 0x110000; ++c) out->cls_packed[c >> 4] |= (uint32_t)cls[c] << ((c & 15) * 2);
  }
  std::unordered_map<std::string, uint32_t> vocab;
  vocab.reserve((size_t)n_vocab * 2);
  for (uint32_t i = 0; i < n_vocab; ++i) {
    // the page kernels keep (id, length) of a token in one 32-bit word: 20 bits of id (model_kernels.cuh tok_pack)
    if (vocab_ids[i] >= (1u << 20)) return "token ids of 2^20 and above are not supported";
    vocab[std::string((const char*)vocab_bytes + vocab_off[i], vocab_off[i + 1] - vocab_off[i])] = vocab_ids[i];
  }
  out->max_chars = max_chars;

  if (model == 0) {
    // ---- ByteLevel alphabet -> ids
    uint32_t cp_of_byte[256];
    bytes_char_table(cp_of_byte);
    std::unordered_map<uint32_t, uint8_t> byte_of_cp;
    out->byte_to_id.assign(256, 0);
    for (int b = 0; b < 256; ++b) {
      std::string ch;
      utf8_append(ch, cp_of_byte[b]);
      auto it = vocab.find(ch);
      if (it == vocab.end())
        return "BPE vocab lacks the ByteLevel character of byte " + std::to_string(b) +
               " (the reference would silently drop such bytes; unsupported on device)";
      out->byte_to_id[b] = it->second;
      byte_of_cp[cp_of_byte[b]] = (uint8_t)b;
    }
    // ---- merges (models/bpe/model.rs:252-275)
    uint32_t cap = pow2_at_least((uint64_t)n_merges * 5 / 2 + 16);
    out->merge_tbl.assign(cap, make_uint4(EMPTY_KEY, EMPTY_KEY, EMPTY_KEY, EMPTY_KEY));
    for (uint32_t i = 0; i < n_merges; ++i) {
      std::string a((const char*)merge_bytes + merge_off[2 * i], merge_off[2 * i + 1] - merge_off[2 * i]);
      std::string b((const char*)merge_bytes + merge_off[2 * i + 1], merge_off[2 * i + 2] - merge_off[2 * i + 1]);
      auto ia = vocab.find(a), ib = vocab.find(b), in = vocab.find(a + b);
      if (ia == vocab.end() || ib == vocab.end() || in == vocab.end()) {
        *vocab_err = true;
        return "merge " + std::to_string(i) + ": token out of vocabulary";  // Error::MergeTokenOutOfVocabulary
      }
      uint32_t h = pair_hash(ia->second, ib->second) & (cap - 1);
      while (true) {
        uint4& e = out->merge_tbl[h];
        if (e.x == EMPTY_KEY || (e.x == ia->second && e.y == ib->second)) {  // a later duplicate overwrites (HashMap collect)
          e = make_uint4(ia->second, ib->second, i, in->second);
          break;
        }
        h = (h + 1) & (cap - 1);
      }
    }
    // ---- monotonicity: rank of every merge > rank of every merge that creates one of its parts
    {
      std::unordered_map<uint32_t, uint32_t> created;  // token id -> highest rank of a merge producing it
      bool mono = true;
      uint32_t live = 0;
      for (const uint4& e : out->merge_tbl) {
        if (e.x == EMPTY_KEY) continue;
        ++live;
        auto it = created.find(e.w);
        if (it == created.end() || it->second < e.z) created[e.w] = e.z;
      }
      if (live != n_merges) mono = false;  // duplicate pairs were overwritten: be conservative
      for (const uint4& e : out->merge_tbl) {
        if (e.x == EMPTY_KEY) continue;
        auto ia = created.find(e.x), ib = created.find(e.y);
        if ((ia != created.end() && ia->second >= e.z) || (ib != created.end() && ib->second >= e.z)) { mono = false; break; }
      }
      out->monotone = mono;
    }
    // ---- byte pairs that are tokens, byte triples inside tokens (soft cuts of long pre-tokens, long_kernels.cuh)
    {
      out->tok2_bits.assign((1u << 16) / 32, 0u);
      out->tri_bits.assign((1u << 24) / 32, 0u);
      for (uint32_t i = 0; i < n_vocab; ++i) {
        const uint8_t* s = vocab_bytes + vocab_off[i];
        const uint32_t len = vocab_off[i + 1] - vocab_off[i];
        std::vector<uint8_t> raw;
        bool ok = len > 0;
        for (uint32_t p = 0; p < len && ok;) {  // byte-level chars back to bytes
          uint32_t b0 = s[p], cp, l;
          if (b0 < 0x80) { cp = b0; l = 1; }
          else if (b0 < 0xE0 && p + 1 < len) { cp = ((b0 & 31u) << 6) | (s[p + 1] & 63u); l = 2; }
          else { ok = false; break; }
          auto it = byte_of_cp.find(cp);
          if (it == byte_of_cp.end()) { ok = false; break; }
          raw.push_back((uint8_t)it->second);
          p += l;
        }
        if (!ok) continue;  // not a string of ByteLevel characters: no merge can produce it from text
        if (raw.size() == 2) { const uint32_t k = raw[0] | ((uint32_t)raw[1] << 8); out->tok2_bits[k >> 5] |= 1u << (k & 31); }
        for (size_t p = 0; p + 2 < raw.size(); ++p) {
          const uint32_t k = raw[p] | ((uint32_t)raw[p + 1] << 8) | ((uint32_t)raw[p + 2] << 16);
          out->tri_bits[k >> 5] |= 1u << (k & 31);
        }
      }
    }
    // ---- whole-word table for ignore_merges (models/bpe/model.rs:558-567)
    if (ignore_merges) {
      uint32_t wcap = pow2_at_least((uint64_t)n_vocab * 5 / 2 + 16);
      out->word_tbl.assign(wcap, make_uint4(0, 0, EMPTY_KEY, 0));
      for (uint32_t i = 0; i < n_vocab; ++i) {
        const uint8_t* s = vocab_bytes + vocab_off[i];
        uint32_t len = vocab_off[i + 1] - vocab_off[i];
        std::string raw;
        bool ok = len > 0;
        for (uint32_t p = 0; p < len && ok;) {  // byte-level chars back to bytes
          uint32_t b0 = s[p], cp, l;
          if (b0 < 0x80) { cp = b0; l = 1; }
          else if (b0 < 0xE0 && p + 1 < len) { cp = ((b0 & 31u) << 6) | (s[p + 1] & 63u); l = 2; }
          else { ok = false; break; }
          auto it = byte_of_cp.find(cp);
          if (it == byte_of_cp.end()) { ok = false; break; }
          raw.push_back((char)it->second);
          p += l;
        }
        if (!ok) continue;  // contains a char outside the byte alphabet: can never equal a pre-token
        StrHash h;
        strhash_init(h);
        for (unsigned char c : raw) strhash_byte(h, c);
        strhash_fin(h);
        uint32_t slot = h.h1 & (wcap - 1);
        while (out->word_tbl[slot].z != EMPTY_KEY) slot = (slot + 1) & (wcap - 1);
        out->word_tbl[slot] = make_uint4(h.h2, (uint32_t)raw.size(), vocab_ids[i], (uint32_t)out->word_pool.size());
        out->word_pool.insert(out->word_pool.end(), raw.begin(), raw.end());
      }
      out->word_pool.resize(out->word_pool.size() + 16, 0);
    }
  } else {
    // ---- WordPiece: byte trie with two roots
    if (!unk_token) return "WordPiece needs unk_token";
    // the WordPiece page kernel keeps a 416-byte halo: a word of max_input_chars_per_word 4-byte characters must fit it
    // (a longer limit would silently turn long multi-byte words into [UNK])
    if ((uint64_t)max_chars * 4 > 416) return "max_input_chars_per_word above 104 is not supported";
    auto iu = vocab.find(unk_token);
    if (iu == vocab.end()) {
      *vocab_err = true;
      return "WordPiece error: Missing [UNK] token from the vocabulary";  // wordpiece/mod.rs:17-22
    }
    out->unk_id = iu->second;
    std::string prefix = cont_prefix ? cont_prefix : "";
    std::unordered_map<uint64_t, uint32_t> edges;  // node << 8 | byte -> child
    std::vector<uint32_t> node_tok(2, EMPTY_KEY);
    auto insert = [&](uint32_t root, const uint8_t* s, uint32_t len, uint32_t id) {
      uint32_t node = root;
      for (uint32_t p = 0; p < len; ++p) {
        uint64_t key = ((uint64_t)node << 8) | s[p];
        auto it = edges.find(key);
        if (it == edges.end()) {
          uint32_t child = (uint32_t)node_tok.size();
          node_tok.push_back(EMPTY_KEY);
          edges.emplace(key, child);
          node = child;
        } else node = it->second;
      }
      node_tok[node] = id;
    };
    for (uint32_t i = 0; i < n_vocab; ++i) {
      const uint8_t* s = vocab_bytes + vocab_off[i];
      uint32_t len = vocab_off[i + 1] - vocab_off[i];
      if (len == 0) continue;
      insert(0, s, len, vocab_ids[i]);
      if (len > prefix.size() && memcmp(s, prefix.data(), prefix.size()) == 0)
        insert(1, s + prefix.size(), len - (uint32_t)prefix.size(), vocab_ids[i]);
    }
    if (node_tok.size() >= (1u << 24)) return "WordPiece vocabulary too large for the device trie";
    uint32_t ecap = pow2_at_least((uint64_t)edges.size() * 5 / 2 + 16);
    out->edge_tbl.assign(ecap, make_uint4(EMPTY_KEY, 0, EMPTY_KEY, 0));
    for (auto& kv : edges) {
      uint32_t node = (uint32_t)(kv.first >> 8), byte = (uint32_t)(kv.first & 255);
      uint32_t slot = edge_hash(node, byte) & (ecap - 1);
      while (out->edge_tbl[slot].x != EMPTY_KEY) slot = (slot + 1) & (ecap - 1);
      out->edge_tbl[slot] = make_uint4((uint32_t)kv.first, kv.second, node_tok[kv.second], 0);
    }
  }
  return "";
}

}  // namespace b2t

namespace b2t {

// decoders/wordpiece.rs:31-44 cleanup(): the replacements in order, each over the whole string
static void wordpiece_cleanup(std::string& s) {
  static const char* const from_to[][2] = {{" .", "."}, {" ?", "?"}, {" !", "!"}, {" ,", ","}, {" ' ", "'"}, {" n't", "n't"},
                                           {" 'm", "'m"}, {" do not", " don't"}, {" 's", "'s"}, {" 've", "'ve"}, {" 're", "'re"}};
  for (const auto& ft : from_to) {
    const std::string a = ft[0], b = ft[1];
    std::string r;
    size_t i = 0;
    for (size_t j; (j = s.find(a, i)) != std::string::npos; i = j + a.size()) r.append(s, i, j - i).append(b);
    r.append(s, i, std::string::npos);
    s.swap(r);
  }
}

// byte_level.rs:156-171 per token: every char through the inverse byte map, or the token's own UTF-8 when a char is not in it
static std::string bytelevel_image(const std::string& t, const int16_t* byte_of_cp, uint32_t n_cp) {
  std::string r;
  for (size_t i = 0; i < t.size();) {
    const uint8_t b = (uint8_t)t[i];
    const uint32_t n = b < 0x80 ? 1 : (b >> 5) == 6 ? 2 : (b >> 4) == 14 ? 3 : (b >> 3) == 30 ? 4 : 0;
    if (n == 0 || i + n > t.size()) return t;
    uint32_t cp = n == 1 ? b : b & (0x7Fu >> n);
    for (uint32_t k = 1; k < n; ++k) cp = cp << 6 | ((uint8_t)t[i + k] & 63u);
    if (cp >= n_cp || byte_of_cp[cp] < 0) return t;
    r.push_back((char)byte_of_cp[cp]);
    i += n;
  }
  return r;
}

std::string build_decoder_table(int kind, const char* prefix, bool cleanup, bool normalizer, uint32_t n_vocab, const uint8_t* vocab_bytes,
                                const uint32_t* vocab_off, const uint32_t* vocab_ids, uint32_t n_added, const uint8_t* added_bytes,
                                const uint32_t* added_off, const uint32_t* added_ids, const uint8_t* added_flags, DecoderHost* out) {
  if (kind != B2T_DECODER_NONE && kind != B2T_DECODER_BYTELEVEL && kind != B2T_DECODER_WORDPIECE) return "decoder kind " + std::to_string(kind) + " is not supported on the device";
  // id -> string: the model's, then the added vocabulary's over it
  uint32_t n_ids = 0;
  for (uint32_t i = 0; i < n_vocab; ++i) n_ids = std::max(n_ids, vocab_ids[i] + 1);
  for (uint32_t i = 0; i < n_added; ++i) n_ids = std::max(n_ids, added_ids[i] + 1);
  for (uint32_t i = 0; i < n_vocab; ++i) if (vocab_ids[i] >= DEC_MAX_IDS) return "vocabulary id " + std::to_string(vocab_ids[i]) + ": ids of 2^20 and above are not supported";
  for (uint32_t i = 0; i < n_added; ++i) if (added_ids[i] >= DEC_MAX_IDS) return "added token id " + std::to_string(added_ids[i]) + ": ids of 2^20 and above are not supported";
  std::vector<const uint8_t*> str(n_ids, nullptr);
  std::vector<uint32_t> len(n_ids, 0);
  for (uint32_t i = 0; i < n_vocab; ++i) { str[vocab_ids[i]] = vocab_bytes + vocab_off[i]; len[vocab_ids[i]] = vocab_off[i + 1] - vocab_off[i]; }
  std::unordered_map<std::string, bool> special;
  for (uint32_t i = 0; i < n_added; ++i) {
    if (normalizer && (added_flags[i] & B2T_ADDED_NORMALIZED))
      return "added tokens with normalized=true behind a normalizer: their decoded string is not settled (the normalized form or the content)";
    str[added_ids[i]] = added_bytes + added_off[i]; len[added_ids[i]] = added_off[i + 1] - added_off[i];
    if (added_flags[i] & B2T_ADDED_SPECIAL) special[std::string((const char*)added_bytes + added_off[i], added_off[i + 1] - added_off[i])] = true;
  }
  int16_t byte_of_cp[0x144];
  std::fill(byte_of_cp, byte_of_cp + 0x144, (int16_t)-1);
  uint32_t cp_of_byte[256];
  bytes_char_table(cp_of_byte);
  for (int b = 0; b < 256; ++b) byte_of_cp[cp_of_byte[b]] = (int16_t)b;
  const std::string pre = prefix ? prefix : "";
  out->ent.assign(n_ids, 0ull);
  out->pool.clear();
  for (uint32_t id = 0; id < n_ids; ++id) {
    if (!str[id]) continue;
    const std::string t((const char*)str[id], len[id]);
    std::string first, rest;
    if (kind == B2T_DECODER_BYTELEVEL) first = rest = bytelevel_image(t, byte_of_cp, 0x144);
    else if (kind == B2T_DECODER_NONE) { first = t; rest = " " + t; }
    else {   // wordpiece.rs:47-61: a later token loses the prefix or gains a space, then cleanup on the token alone
      first = t;
      rest = t.compare(0, pre.size(), pre) == 0 ? t.substr(pre.size()) : " " + t;
      if (cleanup) { wordpiece_cleanup(first); wordpiece_cleanup(rest); }
    }
    if (first.size() > DEC_LEN_MASK || rest.size() > DEC_LEN_MASK) return "token " + std::to_string(id) + ": a decoded image over 16383 bytes is not supported";
    if (out->pool.size() + first.size() + rest.size() >= (1ull << 32)) return "decoder images over 4 GiB are not supported";
    const uint64_t off = out->pool.size();
    out->pool.insert(out->pool.end(), first.begin(), first.end());
    out->pool.insert(out->pool.end(), rest.begin(), rest.end());
    const uint32_t meta = (uint32_t)first.size() | (uint32_t)rest.size() << DEC_LEN_BITS | DEC_EXISTS | (special.count(t) ? DEC_SKIP : 0u);
    out->ent[id] = off | (uint64_t)meta << 32;
  }
  out->pool.resize(out->pool.size() + 16, 0);
  return "";
}

}  // namespace b2t
