// host_tables.h -- host-side construction of the device tables from the engine configuration.
//
// Restates the one-time table building of the reference (paths relative to tokenizers/src of huggingface/tokenizers):
//   pre_tokenizers/byte_level.rs:15-39   bytes_char(): the byte <-> unicode char map of ByteLevel
//   models/bpe/model.rs:252-275          merges (a, b) -> ids through the vocab, new token = a + b
//   models/wordpiece/mod.rs:143-153      vocab, unk token, continuing subword prefix
#pragma once
#include <stdint.h>
#include <string>
#include <unordered_map>
#include <vector>
#include "b2t_tables.h"

namespace b2t {

struct HostTables {
  std::vector<uint32_t> cls_packed;   // 2 bits per code point
  std::vector<uint32_t> byte_to_id;   // 256
  std::vector<uint4> merge_tbl;
  std::vector<uint4> word_tbl;
  std::vector<uint8_t> word_pool;
  std::vector<uint4> edge_tbl;
  // BPE: which byte pairs are 2-byte tokens / which byte triples occur inside some token (raw bytes): a token can only
  // span a byte boundary whose pair / triples pass these tests, everywhere else a long pre-token can be cut exactly
  std::vector<uint32_t> tok2_bits;    // 2^16 bits
  std::vector<uint32_t> tri_bits;     // 2^24 bits
  uint32_t unk_id = EMPTY_KEY;
  uint32_t max_chars = 100;
  bool monotone = false;
};

// BertNormalizer as a per-code-point table (norm_kernels.cuh NormTables)
struct NormHost {
  std::vector<uint16_t> blk;
  std::vector<uint32_t> ent;
  std::vector<uint8_t> pool;
  std::vector<uint8_t> ascii;
  bool ok = true;   // every image fits the kernels' bound of 3 bytes per input byte
};
void build_bert_norm(bool clean_text, bool handle_chinese_chars, bool strip_accents, bool lowercase, NormHost* out);

// Fills out[0x110000] with the class of every code point (scheme 0 = Oniguruma L/N/S, 1 = Rust regex \w,\s,
// 2 = BertPreTokenizer: CLS_S whitespace, CLS_O punctuation, CLS_L everything else).
void unicode_class_table(int scheme, uint8_t* out);

// A token string as ByteLevel::process_offsets (pre_tokenizers/byte_level.rs:202-234) counts it: its chars, and its
// leading / trailing chars that are U+0120 or whitespace (cls: scheme 1 of unicode_class_table, \s = CLS_S).
void space_counts(const uint8_t* s, uint32_t len, const uint8_t* cls, uint32_t* chars, uint32_t* lead, uint32_t* trail);

// Per vocabulary id (ids above the largest are not in the table): space_counts' lead | trail << 16 of its string.
std::vector<uint32_t> vocab_trim_counts(uint32_t n_vocab, const uint8_t* vocab_bytes, const uint32_t* vocab_off, const uint32_t* vocab_ids);

// The decoder table (b2t_tables.h DEC_*): entry per id in [0, largest id], images back to back in pool.  kind: 0 none, 1
// ByteLevel, 2 WordPiece.  The added vocabulary wins over the model's (added_vocabulary.rs simple_id_to_token); a special
// added token's content marks every id with that string.  Returns "" on success, else the reason for B2T_ERR_UNSUPPORTED.
struct DecoderHost {
  std::vector<uint64_t> ent;
  std::vector<uint8_t> pool;
};
std::string build_decoder_table(int kind, const char* prefix, bool cleanup, bool normalizer, uint32_t n_vocab, const uint8_t* vocab_bytes,
                                const uint32_t* vocab_off, const uint32_t* vocab_ids, uint32_t n_added, const uint8_t* added_bytes,
                                const uint32_t* added_off, const uint32_t* added_ids, const uint8_t* added_flags, DecoderHost* out);

// Returns "" on success, else an error message; *vocab_err distinguishes B2T_ERR_VOCAB from B2T_ERR_UNSUPPORTED.
std::string build_host_tables(int model, int pretok, int ignore_merges, uint32_t n_vocab, const uint8_t* vocab_bytes,
                              const uint32_t* vocab_off, const uint32_t* vocab_ids, uint32_t n_merges,
                              const uint8_t* merge_bytes, const uint32_t* merge_off, const char* unk_token,
                              const char* cont_prefix, uint32_t max_chars, HostTables* out, bool* vocab_err);

}  // namespace b2t
