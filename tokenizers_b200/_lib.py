"""ctypes binding of libb2t.so (include/b2t.h).  There is no Python/CPU fallback: a missing library is an error."""
import ctypes, os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2T_LIB") or os.path.join(_HERE, "libb2t.so")  # B2T_LIB: developer override for A/B builds

B2T_OK, B2T_ERR_INVALID, B2T_ERR_UNSUPPORTED, B2T_ERR_CUDA, B2T_ERR_VOCAB, B2T_ERR_TOO_LARGE, B2T_ERR_TRUNCATION = range(7)
MODEL_BPE, MODEL_WORDPIECE = 0, 1
PRETOK_BYTELEVEL, PRETOK_LLAMA3, PRETOK_WHITESPACE, PRETOK_BYTELEVEL_NOREGEX, PRETOK_BERT = 0, 1, 2, 3, 4
NORM_BERT, NORM_CLEAN_TEXT, NORM_CHINESE_CHARS, NORM_STRIP_ACCENTS, NORM_LOWERCASE = 0x100, 1, 2, 4, 8
WANT_OFFSETS, WANT_WORD_IDS, OFFSETS_BYTES, NO_ADDED_TOKENS, FLAG_ADDED_IDS = 1, 2, 4, 8, 16
ADDED_SINGLE_WORD, ADDED_LSTRIP, ADDED_RSTRIP, ADDED_NORMALIZED = 1, 2, 4, 8
TRUNC_LONGEST_FIRST, TRUNC_ONLY_FIRST, TRUNC_ONLY_SECOND = 0, 1, 2
PIECE_A, PIECE_B = 0x80000000, 0x80000001
DENSE_OVERFLOW, DENSE_OFFSETS = 1, 2
DENSE_TRIM_OFFSETS, DENSE_TRIM_PREFIX_SPACE, DENSE_SPECIAL_MASK, DENSE_SEQUENCE_IDS, DENSE_WORD_IDS = 4, 8, 16, 32, 64
DECODER_NONE, DECODER_BYTELEVEL, DECODER_WORDPIECE = 0, 1, 2
ADDED_SPECIAL = 16
DECODE_SKIP_SPECIAL = 1

# every symbol include/b2t.h declares
SYMBOLS = ["b2t_engine_create", "b2t_engine_destroy", "b2t_engine_set_added_tokens", "b2t_encode_batch", "b2t_encode_batch_device", "b2t_encode_batch_device_begin",
           "b2t_encode_batch_device_finish", "b2t_pre_tokenize_batch",
           "b2t_encode_batch_dense", "b2t_encode_batch_dense_device", "b2t_result_dense_length", "b2t_result_dense_ids",
           "b2t_result_attention_mask", "b2t_result_row_lengths",
           "b2t_encode_pairs_dense", "b2t_encode_pairs_dense_device", "b2t_result_type_ids",
           "b2t_result_dense_rows", "b2t_result_row_sample", "b2t_result_dense_offsets",
           "b2t_result_special_tokens_mask", "b2t_result_sequence_ids", "b2t_result_dense_word_ids",
           "b2t_result_n_tokens", "b2t_result_n_docs", "b2t_result_on_device", "b2t_result_ids", "b2t_result_offsets",
           "b2t_result_word_ids", "b2t_result_row_ptr", "b2t_result_free", "b2t_host_alloc", "b2t_host_free",
           "b2t_engine_set_profiling", "b2t_engine_last_kernels", "b2t_unicode_class_table", "b2t_bert_normalizer_images", "b2t_last_error", "b2t_version",
           "b2t_engine_set_decoder", "b2t_decoder_images", "b2t_decode_batch", "b2t_decode_batch_device", "b2t_result_text", "b2t_result_text_off"]


class Config(ctypes.Structure):
    _fields_ = [("struct_size", ctypes.c_uint32), ("model", ctypes.c_int32), ("pretok", ctypes.c_int32),
                ("add_prefix_space", ctypes.c_int32), ("ignore_merges", ctypes.c_int32),
                ("n_vocab", ctypes.c_uint32), ("vocab_bytes", ctypes.c_void_p), ("vocab_off", ctypes.c_void_p),
                ("vocab_ids", ctypes.c_void_p),
                ("n_merges", ctypes.c_uint32), ("merge_bytes", ctypes.c_void_p), ("merge_off", ctypes.c_void_p),
                ("unk_token", ctypes.c_char_p), ("continuing_subword_prefix", ctypes.c_char_p),
                ("max_input_chars_per_word", ctypes.c_uint32), ("device", ctypes.c_int32), ("bert_normalizer", ctypes.c_int32)]


class DenseSpec(ctypes.Structure):
    _fields_ = [("struct_size", ctypes.c_uint32), ("length", ctypes.c_uint32), ("pad_to_multiple_of", ctypes.c_uint32),
                ("max_length", ctypes.c_uint32), ("pad_id", ctypes.c_uint32), ("truncate_left", ctypes.c_int32), ("pad_left", ctypes.c_int32),
                ("n_pre", ctypes.c_uint32), ("n_post", ctypes.c_uint32), ("pre_ids", ctypes.c_void_p), ("post_ids", ctypes.c_void_p),
                ("want_mask", ctypes.c_uint32), ("stride", ctypes.c_uint32), ("dense_flags", ctypes.c_uint32)]


class PairDenseSpec(ctypes.Structure):
    _fields_ = [("struct_size", ctypes.c_uint32), ("length", ctypes.c_uint32), ("pad_to_multiple_of", ctypes.c_uint32),
                ("max_length", ctypes.c_uint32), ("strategy", ctypes.c_int32), ("truncate_left", ctypes.c_int32),
                ("pad_id", ctypes.c_uint32), ("pad_type_id", ctypes.c_uint32), ("pad_left", ctypes.c_int32),
                ("n_pieces", ctypes.c_uint32), ("piece_ids", ctypes.c_void_p), ("piece_types", ctypes.c_void_p),
                ("want_mask", ctypes.c_uint32), ("stride", ctypes.c_uint32), ("dense_flags", ctypes.c_uint32),
                ("overflow_type_a", ctypes.c_uint32), ("overflow_type_b", ctypes.c_uint32)]

class DecoderSpec(ctypes.Structure):
    _fields_ = [("struct_size", ctypes.c_uint32), ("kind", ctypes.c_int32), ("prefix", ctypes.c_char_p), ("cleanup", ctypes.c_int32),
                ("n_added", ctypes.c_uint32), ("added_bytes", ctypes.c_void_p), ("added_off", ctypes.c_void_p), ("added_ids", ctypes.c_void_p),
                ("added_flags", ctypes.c_void_p)]

# the specs' size before stride and dense_flags were appended (accepted by the engine: those fields read as 0)
DENSE_SPEC_V1_SIZE = PAIR_DENSE_SPEC_V1_SIZE = 64


class B2TError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(msg)
        self.code = code


_lib = None


def lib():
    """Load libb2t.so (built by tokenizers_b200/csrc/Makefile or __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `make -C tokenizers_b200/csrc` "
                          "(there is no fallback implementation)")
    L = ctypes.CDLL(LIB_PATH)
    vp, u32, u64, i32 = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int
    L.b2t_engine_create.argtypes = [ctypes.POINTER(Config), ctypes.POINTER(vp)]
    L.b2t_engine_destroy.argtypes = [vp]; L.b2t_engine_destroy.restype = None
    L.b2t_engine_set_added_tokens.argtypes = [vp, u32, vp, vp, vp, vp]
    L.b2t_encode_batch.argtypes = [vp, vp, vp, u32, u32, ctypes.POINTER(vp)]
    L.b2t_encode_batch_device.argtypes = [vp, vp, u64, vp, u32, u32, vp, ctypes.POINTER(vp)]
    L.b2t_encode_batch_device_begin.argtypes = [vp, vp, u64, vp, u32, u32, vp, ctypes.POINTER(u64)]
    L.b2t_encode_batch_device_finish.argtypes = [vp, vp, vp, vp, vp, u64, vp]
    L.b2t_pre_tokenize_batch.argtypes = [vp, vp, vp, u32, ctypes.POINTER(vp)]
    L.b2t_encode_batch_dense.argtypes = [vp, vp, vp, u32, ctypes.POINTER(DenseSpec), ctypes.POINTER(vp)]
    L.b2t_encode_batch_dense_device.argtypes = [vp, vp, u64, vp, u32, ctypes.POINTER(DenseSpec), vp, ctypes.POINTER(vp)]
    L.b2t_result_dense_length.argtypes = [vp]; L.b2t_result_dense_length.restype = u32
    L.b2t_encode_pairs_dense.argtypes = [vp, vp, vp, u32, ctypes.POINTER(PairDenseSpec), ctypes.POINTER(vp)]
    L.b2t_encode_pairs_dense_device.argtypes = [vp, vp, u64, vp, u32, ctypes.POINTER(PairDenseSpec), vp, ctypes.POINTER(vp)]
    L.b2t_result_dense_rows.argtypes = [vp]; L.b2t_result_dense_rows.restype = u32
    for f in ("b2t_result_dense_ids", "b2t_result_attention_mask", "b2t_result_row_lengths", "b2t_result_type_ids", "b2t_result_row_sample",
              "b2t_result_dense_offsets", "b2t_result_special_tokens_mask", "b2t_result_sequence_ids", "b2t_result_dense_word_ids"):
        getattr(L, f).argtypes = [vp]; getattr(L, f).restype = vp
    L.b2t_result_n_tokens.argtypes = [vp]; L.b2t_result_n_tokens.restype = u64
    L.b2t_result_n_docs.argtypes = [vp]; L.b2t_result_n_docs.restype = u32
    L.b2t_result_on_device.argtypes = [vp]; L.b2t_result_on_device.restype = i32
    for f in ("b2t_result_ids", "b2t_result_offsets", "b2t_result_word_ids", "b2t_result_row_ptr"):
        getattr(L, f).argtypes = [vp]; getattr(L, f).restype = vp
    L.b2t_result_free.argtypes = [vp]; L.b2t_result_free.restype = None
    L.b2t_host_alloc.argtypes = [ctypes.c_size_t, ctypes.POINTER(vp)]
    L.b2t_host_free.argtypes = [vp]; L.b2t_host_free.restype = None
    L.b2t_engine_set_profiling.argtypes = [vp, i32]
    L.b2t_engine_last_kernels.argtypes = [vp, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_float), i32]
    L.b2t_unicode_class_table.argtypes = [i32, vp]
    L.b2t_bert_normalizer_images.argtypes = [i32, vp, ctypes.c_size_t, vp]
    L.b2t_engine_set_decoder.argtypes = [vp, ctypes.POINTER(DecoderSpec)]
    L.b2t_decoder_images.argtypes = [ctypes.POINTER(Config), ctypes.POINTER(DecoderSpec), vp, vp, ctypes.POINTER(u32), ctypes.POINTER(u64)]
    L.b2t_decode_batch.argtypes = [vp, vp, u64, vp, vp, u32, u32, ctypes.POINTER(vp)]
    L.b2t_decode_batch_device.argtypes = [vp, vp, u64, vp, vp, u32, u32, vp, ctypes.POINTER(vp)]
    for f in ("b2t_result_text", "b2t_result_text_off"):
        getattr(L, f).argtypes = [vp]; getattr(L, f).restype = vp
    L.b2t_last_error.restype = ctypes.c_char_p
    L.b2t_version.restype = ctypes.c_char_p
    _lib = L
    return L


def check(rc):
    if rc != B2T_OK:
        raise B2TError(rc, lib().b2t_last_error().decode("utf-8", "replace"))
