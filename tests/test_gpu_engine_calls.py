"""GPU (-m gpu): the host-side call paths of the engine (csrc/engine.cu) that the encode tests do not reach on their own:
the rerun with a grown long pool at every entry point, the begin / finish split of the device-resident entry point on
one GPU, the per-kernel profiling record, and the argument checks of the host-buffer and device-resident entry points."""
import ctypes
import numpy as np
import pytest
import helpers, corpus

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402

FLAGS = 1 | 2   # WANT_OFFSETS | WANT_WORD_IDS


def lib():
    from tokenizers_b200 import _lib
    return _lib, _lib.lib()


def on_device(data, off):
    import torch
    return (torch.from_numpy(np.concatenate([np.asarray(data, dtype=np.uint8), np.zeros(64, np.uint8)])).cuda(),
            torch.from_numpy(np.asarray(off).astype(np.int64)).cuda())


def copy_back(ptr, count, dtype):
    out = np.empty(count, dtype=dtype)
    if count:
        assert ctypes.CDLL("libcudart.so").cudaMemcpy(ctypes.c_void_p(out.ctypes.data), ctypes.c_void_p(ptr), ctypes.c_size_t(out.nbytes), 2) == 0
    return out


# ---------------------------------------------------------------------------------------------- long-pool rerun
# The BPE pre-pass for long pre-tokens (csrc/long_kernels.cuh) places every piece that is still longer than 256 bytes
# after the soft cuts in a pool that starts at (1 << 20) * 5 / 4 + 4096 = 1,314,816 bytes per workspace.  A run of one
# letter whose doubled form is a vocabulary token ("oo", "ee", "ss" in the gpt2_style asset) cannot be cut anywhere: the
# pair at every boundary is a token.  So each of these documents is one long pre-token of ~70 KB, and a batch of more
# than ~19 of them overflows the pool: the engine grows it to what the run asked for and runs the batch again.
LONG_BASE = ["o" * 70000, "e" * 70001, "s" * 69999 + " so", "x " * 40]


def long_batch(target_bytes, seed):
    base_data, base_off = helpers.pack_docs(LONG_BASE)
    data, off, shims = helpers.tiled_batch(base_data, base_off, target_bytes, seed=seed)
    return data, off, base_data, base_off, shims


def long_expectation(o, base_data, base_off, shims):
    return helpers.tiled_expectation(lambda d, f: o.encode_batch_csr(d, f), base_data, base_off, shims)


def test_long_pool_rerun_host_chunks():
    """b2t_encode_batch in 2 MiB chunks (over 2 MB of long pre-tokens each, so every chunk alone overflows its slot's
    pool), 5+ chunks: the first chunk of each of the three slots reruns in drain while other chunks are in flight"""
    tj = helpers.asset_json("gpt2_style")
    data, off, bd, bo, shims = long_batch(10 << 20, seed=1)
    tok = helpers.tokenizer_with_env(tj, B2T_CHUNK_BYTES=2 << 20)
    be = tok.encode_batch_csr(data, off)
    helpers.assert_csr_equal((be.ids, be.offsets, be.word_ids, be.row_ptr), long_expectation(orc.Oracle(tj), bd, bo, shims), None, "host chunks")


@pytest.mark.parametrize("length", [64, None])
def test_long_pool_rerun_host_dense(length):
    """b2t_encode_batch_dense, one chunk: a fixed length (the rows queued right behind the first run are copied again
    after the rerun) and BatchLongest"""
    from tokenizers_b200 import Tokenizer
    tj = helpers.asset_json("gpt2_style")
    data, off, bd, bo, shims = long_batch(3 << 20, seed=2)
    ids, _, _, rp = long_expectation(orc.Oracle(tj), bd, bo, shims)
    tok = Tokenizer.from_str(tj)
    tok.enable_truncation(100 if length is None else length)
    tok.enable_padding(length=length, pad_id=7)
    got = tok.encode_batch_dense(data, off, add_special_tokens=False)
    exp = orc.dense_rows(ids, rp, length=length or 0, pad_to_multiple_of=0, max_length=100 if length is None else length, pad_id=7,
                         truncate_left=False, pad_left=False, pre=[], post=[])
    assert np.array_equal(got["input_ids"], exp[0]) and np.array_equal(got["attention_mask"], exp[1]) and np.array_equal(got["lengths"], exp[2])


def test_long_pool_rerun_device():
    """b2t_encode_batch_device"""
    from tokenizers_b200 import Tokenizer
    tj = helpers.asset_json("gpt2_style")
    data, off, bd, bo, shims = long_batch(3 << 20, seed=3)
    got = helpers.device_csr(Tokenizer.from_str(tj), data, off, FLAGS)
    helpers.assert_csr_equal(got, long_expectation(orc.Oracle(tj), bd, bo, shims), None, "device entry point")


@pytest.mark.parametrize("length", [64, None])
def test_long_pool_rerun_dense_device(length):
    """b2t_encode_batch_dense_device, a fixed length and BatchLongest"""
    from tokenizers_b200 import Tokenizer
    import torch
    _lib, L = lib()
    tj = helpers.asset_json("gpt2_style")
    data, off, bd, bo, shims = long_batch(3 << 20, seed=4)
    ids, _, _, rp = long_expectation(orc.Oracle(tj), bd, bo, shims)
    max_length = 100 if length is None else length
    exp = orc.dense_rows(ids, rp, length=length or 0, pad_to_multiple_of=0, max_length=max_length, pad_id=7, truncate_left=False, pad_left=False,
                         pre=[], post=[])
    tok = Tokenizer.from_str(tj)
    tok.enable_truncation(max_length)
    tok.enable_padding(length=length, pad_id=7)
    sp, keep = tok.dense_spec(add_special_tokens=False)
    d_bytes, d_off = on_device(data, off)
    n = len(off) - 1
    res = ctypes.c_void_p()
    _lib.check(L.b2t_encode_batch_dense_device(tok.handle, d_bytes.data_ptr(), len(data), d_off.data_ptr(), n, ctypes.byref(sp), None, ctypes.byref(res)))
    try:
        torch.cuda.synchronize()
        W = L.b2t_result_dense_length(res)
        assert W == exp[0].shape[1]
        assert np.array_equal(copy_back(L.b2t_result_dense_ids(res), n * W, np.uint32).reshape(n, W), exp[0])
        assert np.array_equal(copy_back(L.b2t_result_attention_mask(res), n * W, np.uint8).reshape(n, W), exp[1])
        assert np.array_equal(copy_back(L.b2t_result_row_lengths(res), n, np.uint32), exp[2])
    finally:
        L.b2t_result_free(res)
    del keep


# ---------------------------------------------------------------------------------------------- begin / finish
def test_begin_finish_into_caller_buffers():
    """b2t_encode_batch_device_begin, then _finish into torch buffers at a token and a row displacement with a token base:
    the CSR of b2t_encode_batch_device, shifted, and nothing written outside it"""
    from tokenizers_b200 import Tokenizer
    import torch
    _lib, L = lib()
    tok = Tokenizer.from_str(helpers.asset_json("gpt2_style"))
    data, off = corpus.generate(2, 41, 0, 3000)
    exp = helpers.device_csr(tok, data, off, FLAGS)
    n, T = len(off) - 1, len(exp[0])
    d_bytes, d_off = on_device(data, off)
    n_tok = ctypes.c_uint64()
    _lib.check(L.b2t_encode_batch_device_begin(tok.handle, d_bytes.data_ptr(), len(data), d_off.data_ptr(), n, FLAGS, None, ctypes.byref(n_tok)))
    assert n_tok.value == T
    td, rd, base = 1000, 7, 123456
    ids = torch.full((T + 2 * td,), -1, dtype=torch.int32, device="cuda")
    offs = torch.full((2 * (T + 2 * td),), -1, dtype=torch.int32, device="cuda")
    wid = torch.full((T + 2 * td,), -1, dtype=torch.int32, device="cuda")
    rp = torch.full((n + 1 + 2 * rd,), -1, dtype=torch.int64, device="cuda")
    _lib.check(L.b2t_encode_batch_device_finish(tok.handle, ids.data_ptr() + 4 * td, offs.data_ptr() + 8 * td, wid.data_ptr() + 4 * td,
                                                rp.data_ptr() + 8 * rd, base, None))
    torch.cuda.synchronize()
    ids, offs, wid, rp = (t.cpu().numpy() for t in (ids, offs, wid, rp))
    assert np.array_equal(ids[td:td + T].view(np.uint32), exp[0])
    assert np.array_equal(offs[2 * td:2 * (td + T)].view(np.uint32).reshape(-1, 2), exp[1])
    assert np.array_equal(wid[td:td + T].view(np.uint32), exp[2])
    assert np.array_equal(rp[rd:rd + n + 1].view(np.uint64), exp[3] + np.uint64(base))
    for outside in (ids[:td], ids[td + T:], offs[:2 * td], offs[2 * (td + T):], wid[:td], wid[td + T:], rp[:rd], rp[rd + n + 1:]):
        assert (outside == -1).all()


def test_finish_refusals():
    """_finish without a begin, and a null d_offsets when offsets were requested at begin: B2T_ERR_INVALID"""
    from tokenizers_b200 import Tokenizer
    import torch
    _lib, L = lib()
    tok = Tokenizer.from_str(helpers.asset_json("gpt2_style"))
    buf = torch.zeros(1 << 16, dtype=torch.int64, device="cuda")
    p = buf.data_ptr()
    assert L.b2t_encode_batch_device_finish(tok.handle, p, p, p, p, 0, None) == _lib.B2T_ERR_INVALID
    data, off = corpus.generate(2, 42, 0, 50)
    d_bytes, d_off = on_device(data, off)
    n_tok = ctypes.c_uint64()
    _lib.check(L.b2t_encode_batch_device_begin(tok.handle, d_bytes.data_ptr(), len(data), d_off.data_ptr(), len(off) - 1, FLAGS, None,
                                               ctypes.byref(n_tok)))
    assert L.b2t_encode_batch_device_finish(tok.handle, p, None, p, p, 0, None) == _lib.B2T_ERR_INVALID
    assert b"d_offsets is null" in L.b2t_last_error()


# ---------------------------------------------------------------------------------------------- profiling record
# Kernel names and launch count of one call with profiling on (what bench.py reports).  The count leaves out the four
# prefix re-pack launches of add_prefix_space, the chunk rebase of the host path and N3 (offsets mapped back behind the
# normalizer).
BPE = ["doc_mark", "pretok_scan", "page_scan", "long_find", "bpe_long", "bpe_tile", "scan_compact"]
PROFILES = {
    "gpt2_style": (BPE, 13),
    "gpt2_prefix": (BPE, 13),
    "llama3_style": (BPE, 13),
    "added_wordpiece": (["doc_mark", "added_tokens", "pretok_scan", "page_scan", "wordpiece_tile", "scan_compact"], 11),
    "bert_uncased": (["normalize", "doc_mark", "pretok_scan", "page_scan", "wordpiece_tile", "scan_compact"], 16),
}


def last_kernels(L, tok):
    names, ms = (ctypes.c_char_p * 16)(), (ctypes.c_float * 16)()
    n = L.b2t_engine_last_kernels(tok.handle, names, ms, 16)
    return [names[i].decode() for i in range(16) if names[i] is not None], n


@pytest.mark.parametrize("name", list(PROFILES))
def test_profiling_record_device(name):
    from tokenizers_b200 import Tokenizer
    _lib, L = lib()
    tok = Tokenizer.from_str(helpers.pipeline_json(name))
    if name.startswith("added_"):
        assert tok._dev_added
        data, off = helpers.pack_docs(helpers.added_token_docs(7, 300))
        flags = FLAGS | _lib.FLAG_ADDED_IDS
    else:
        data, off = corpus.generate(2, 43, 0, 500)
        flags = FLAGS
    _lib.check(L.b2t_engine_set_profiling(tok.handle, 1))
    helpers.device_csr(tok, data, off, flags)
    assert last_kernels(L, tok) == PROFILES[name]


@pytest.mark.parametrize("length", [64, None])
def test_profiling_record_dense_device(length):
    from tokenizers_b200 import Tokenizer
    _lib, L = lib()
    tok = Tokenizer.from_str(helpers.asset_json("gpt2_style"))
    tok.enable_truncation(64)
    tok.enable_padding(length=length)
    sp, keep = tok.dense_spec(add_special_tokens=False)
    data, off = corpus.generate(2, 44, 0, 500)
    d_bytes, d_off = on_device(data, off)
    _lib.check(L.b2t_engine_set_profiling(tok.handle, 1))
    res = ctypes.c_void_p()
    _lib.check(L.b2t_encode_batch_dense_device(tok.handle, d_bytes.data_ptr(), len(data), d_off.data_ptr(), len(off) - 1, ctypes.byref(sp), None,
                                               ctypes.byref(res)))
    L.b2t_result_free(res)
    assert last_kernels(L, tok) == (BPE + ["dense_rows"], 15)
    del keep


# ---------------------------------------------------------------------------------------------- argument checks
BAD_DOC_OFF = [(np.array([1, 11, 18], dtype=np.uint64), b"doc_off[0] must be 0"),
               (np.array([0, 11, 5, 18], dtype=np.uint64), b"non-decreasing")]


@pytest.mark.parametrize("entry", ["b2t_encode_batch", "b2t_encode_batch_dense", "b2t_pre_tokenize_batch"])
def test_host_entry_points_refuse_bad_doc_off(entry):
    from tokenizers_b200 import Tokenizer
    _lib, L = lib()
    tok = Tokenizer.from_str(helpers.asset_json("gpt2_style"))
    tok.enable_padding(length=16)
    sp, keep = tok.dense_spec(add_special_tokens=False)
    data = np.frombuffer(b"hello world, hello", dtype=np.uint8)
    for off, msg in BAD_DOC_OFF:
        res = ctypes.c_void_p()
        n = len(off) - 1
        if entry == "b2t_encode_batch":
            rc = L.b2t_encode_batch(tok.handle, data.ctypes.data, off.ctypes.data, n, FLAGS, ctypes.byref(res))
        elif entry == "b2t_encode_batch_dense":
            rc = L.b2t_encode_batch_dense(tok.handle, data.ctypes.data, off.ctypes.data, n, ctypes.byref(sp), ctypes.byref(res))
        else:
            rc = L.b2t_pre_tokenize_batch(tok.handle, data.ctypes.data, off.ctypes.data, n, ctypes.byref(res))
        assert rc == _lib.B2T_ERR_INVALID and msg in L.b2t_last_error(), (entry, off)
    del keep


@pytest.mark.parametrize("entry", ["b2t_encode_batch_device", "b2t_encode_batch_device_begin", "b2t_encode_batch_dense_device"])
def test_device_entry_points_refuse_misaligned_bytes(entry):
    from tokenizers_b200 import Tokenizer
    _lib, L = lib()
    tok = Tokenizer.from_str(helpers.asset_json("gpt2_style"))
    tok.enable_padding(length=16)
    sp, keep = tok.dense_spec(add_special_tokens=False)
    data, off = corpus.generate(2, 45, 0, 20)
    d_bytes, d_off = on_device(data, off)
    args = (tok.handle, d_bytes.data_ptr() + 1, len(data), d_off.data_ptr(), len(off) - 1)
    res, n_tok = ctypes.c_void_p(), ctypes.c_uint64()
    if entry == "b2t_encode_batch_device":
        rc = L.b2t_encode_batch_device(*args, FLAGS, None, ctypes.byref(res))
    elif entry == "b2t_encode_batch_device_begin":
        rc = L.b2t_encode_batch_device_begin(*args, FLAGS, None, ctypes.byref(n_tok))
    else:
        rc = L.b2t_encode_batch_dense_device(*args, ctypes.byref(sp), None, ctypes.byref(res))
    assert rc == _lib.B2T_ERR_INVALID and b"16-byte aligned" in L.b2t_last_error()
    del keep
