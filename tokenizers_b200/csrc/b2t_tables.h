// b2t_tables.h -- device table layouts and the hash functions shared by the host builders and the kernels.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2T_HDI __host__ __device__ __forceinline__
#else
#define B2T_HDI inline
#endif

namespace b2t {

constexpr uint32_t EMPTY_KEY = 0xFFFFFFFFu;
constexpr uint64_t NO_MERGE = ~0ull;

// (left id, right id) -> slot hash of the merge table (models/bpe/model.rs:22 MergeMap)
B2T_HDI uint32_t pair_hash(uint32_t a, uint32_t b) {
  uint32_t h = a * 0x9E3779B1u ^ (b * 0x85EBCA77u + 0x165667B1u);
  h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
  return h;
}

// byte-string hash (whole-word vocab lookup for ignore_merges): two 32-bit lanes (slot, fingerprint)
struct StrHash {
  uint32_t h1, h2;
};
B2T_HDI void strhash_init(StrHash& s) { s.h1 = 0x811C9DC5u; s.h2 = 0x9747B28Cu; }
B2T_HDI void strhash_byte(StrHash& s, uint32_t b) {
  s.h1 = (s.h1 ^ b) * 0x01000193u;
  s.h2 = (s.h2 + b + 1u) * 0x5BD1E995u; s.h2 ^= s.h2 >> 13;
}
B2T_HDI void strhash_fin(StrHash& s) {
  s.h1 ^= s.h1 >> 16; s.h1 *= 0x7FEB352Du; s.h1 ^= s.h1 >> 15;
  s.h2 ^= s.h2 >> 15; s.h2 *= 0x846CA68Bu; s.h2 ^= s.h2 >> 16;
}

// WordPiece trie edge hash: (node, byte) -> slot
B2T_HDI uint32_t edge_hash(uint32_t node, uint32_t byte) {
  uint32_t h = (node * 256u + byte) * 0x9E3779B1u;
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13;
  return h;
}

// Decoder table (decode_kernels.cuh DecodeTable, include/b2t.h b2t_decoder_images): one entry per id, x = offset of the id's
// images in the pool, y = first image's length | later image's length << 14 | DEC_EXISTS | DEC_SKIP; the later image's
// bytes follow the first image's
constexpr uint32_t DEC_LEN_BITS = 14, DEC_LEN_MASK = (1u << DEC_LEN_BITS) - 1u;
constexpr uint32_t DEC_EXISTS = 1u << 28;   // the id has a string (added vocabulary or model)
constexpr uint32_t DEC_SKIP = 1u << 29;     // its string is the content of a special added token: skip_special_tokens drops it
constexpr uint32_t DEC_MAX_IDS = 1u << 20;

// BertNormalizer table entries (norm_kernels.cuh NormTables.ent): kind in bits 0-1
enum { NORM_IDENT = 0u, NORM_REMOVE = 1u, NORM_STRING = 2u, NORM_SURVIVOR = 3u, NORM_MARK_FLAG = 4u, NORM_TAIL_FLAG = 0x80u };
constexpr uint32_t NORM_LEN_MASK = 31u;   // NORM_STRING: image bytes in bits 2-6 (at most 12), pool offset in bits 8-31
// NORM_SURVIVOR: a character whose NFD starts with a non-zero canonical combining class and that strip_accents keeps
// (image = itself).  Every other such character is NORM_REMOVE under strip_accents, so an IDENT or STRING character starts
// with a class-0 character: no mark in front of it sorts past it.
// NORM_MARK_FLAG on a NORM_REMOVE entry: canonical ordering sees through the removed character -- its NFD starts with a
// non-zero class, or clean_text removes it before NFD runs and the characters on its two sides meet;
// on a NORM_SURVIVOR entry: its image is not itself (no such character today), always refused.
// NORM_TAIL_FLAG on a NORM_STRING entry: its decomposition keeps a character with a non-zero class behind its first
// (U+1D15E -> U+1D157 U+1D165, 13 musical symbols): a mark right behind it can sort in front of that kept piece, which then
// takes the mark's character.  The kernels check what follows it as they check a survivor's neighbours.

// Can NFD's canonical ordering reach a kept mark across its neighbour cp (entry e; ascii: image of an ASCII character,
// 0xFF = removed, which only clean_text does)?  Any other neighbour behind the mark starts with a class-0 character; any
// other in front of it ends with a class-0 character or with pieces of its decomposition that strip_accents drops (a
// NORM_TAIL_FLAG character checks its own look-ahead).  The mark may sort in front of dropped pieces, but they are not first
// pieces and take no character's alignment in NormalizedString::transform, so it keeps its own and the text is the same.
B2T_HDI bool norm_mark_neighbour(uint32_t cp, uint32_t e, const uint8_t* ascii) {
  if (cp < 128u) return ascii[cp] == 0xFFu;
  const uint32_t kind = e & 3u;
  return kind == NORM_SURVIVOR || (kind == NORM_REMOVE && (e & NORM_MARK_FLAG) != 0u);
}

// Everything the model kernels need, passed by value.
struct DeviceTables {
  // BPE
  const uint32_t* byte_to_id;  // 256: id of the ByteLevel char of each byte (byte_level.rs:15-39 + vocab lookup)
  const uint4* merge_tbl;      // open addressing {a, b, rank, new_id}; a == EMPTY_KEY marks a free slot
  uint32_t merge_mask;         // capacity - 1
  // whole pre-token lookup (ignore_merges): {fingerprint, len, id, pool offset}; id == EMPTY_KEY marks a free slot
  const uint4* word_tbl;
  uint32_t word_mask;
  const uint8_t* word_pool;    // token strings as raw bytes (ByteLevel chars mapped back to bytes)
  int ignore_merges;
  int monotone;                // every merge ranks after all merges creating its parts (long_kernels.cuh)
  const uint32_t* tok2_bits;   // bit (b0 | b1 << 8): the two bytes b0 b1 are a token
  const uint32_t* tri_bits;    // bit (b0 | b1 << 8 | b2 << 16): the bytes b0 b1 b2 occur consecutively inside some token
  // WordPiece: byte trie, two roots (0 = word start, 1 = after the continuing-subword prefix)
  const uint4* edge_tbl;       // {node << 8 | byte, child node, token id of child or EMPTY_KEY, 0}; x == EMPTY_KEY free
  uint32_t edge_mask;
  uint32_t unk_id;
  uint32_t max_chars;
};

}  // namespace b2t
