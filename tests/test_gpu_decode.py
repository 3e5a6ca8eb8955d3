"""GPU: device decode (b2t_decode_batch, b2t_decode_batch_device; Tokenizer.decode_batch_csr / decode_batch_rows) against the
golden fixture of the reference wheel's decode_batch and, where it is importable, the wheel itself: exact strings."""
import gzip, json, os, threading
import numpy as np
import pytest
import helpers
import decode_cases as dc
from tokenizers_b200 import Tokenizer, UnsupportedConfig, B2TError, _lib

pytestmark = pytest.mark.gpu
GOLDEN = dc.load_golden()["configs"]
_TOKS = {}


def tok(name):
    if name not in _TOKS:
        _TOKS[name] = Tokenizer.from_str(dc.tokenizer_json(name), device=0)
    return _TOKS[name]


def csr(rows):
    ids = np.array([i for r in rows for i in r], dtype=np.uint64)
    rp = np.zeros(len(rows) + 1, dtype=np.uint64)
    np.cumsum([len(r) for r in rows], out=rp[1:])
    return ids, rp


def texts(text, off):
    tb, o = text.tobytes(), off.tolist()
    return [tb[o[i]:o[i + 1]].decode("utf-8") for i in range(len(o) - 1)]


def padded(rows, pad=0):
    w = max([len(r) for r in rows] + [1])
    a = np.full((len(rows), w), pad, dtype=np.int64)
    for i, r in enumerate(rows):
        a[i, :len(r)] = r
    return a, np.array([len(r) for r in rows], dtype=np.int64)


def all_paths(t, rows, skip):
    """decode of rows through the host CSR entry point, numpy rows, int32 and int64 CUDA rows (device entry point)"""
    import torch
    ids, rp = csr(rows)
    out = {"csr": texts(*t.decode_batch_csr(ids, rp, skip_special_tokens=skip))}
    a, ln = padded(rows)
    out["numpy"] = t.decode_batch_rows(a, ln, skip_special_tokens=skip)
    out["cuda_int64"] = t.decode_batch_rows(torch.from_numpy(a).cuda(), torch.from_numpy(ln).cuda(), skip_special_tokens=skip)
    a32 = np.minimum(a, (1 << 31) - 1).astype(np.int32)   # (ids of 2^31 and above, unknown, as another unknown id)
    out["cuda_int32"] = t.decode_batch_rows(torch.from_numpy(a32).cuda(), ln, skip_special_tokens=skip)
    return out


@pytest.mark.parametrize("name", list(GOLDEN))
def test_golden_every_entry_point(name):
    g = GOLDEN[name]
    t = tok(name)
    for skip, key in ((True, "skip"), (False, "keep")):
        for path, got in all_paths(t, g["rows"], skip).items():
            assert got == g[key], (name, skip, path, next(i for i in range(len(got)) if got[i] != g[key][i]))


@pytest.mark.parametrize("name", ["gpt2_bytelevel", "llama3_bytelevel", "wordpiece_cleanup", "vocabgen_bpe_high", "vocabgen_wordpiece_high"])
def test_random_ids_over_the_whole_table(name):
    """random ids over [0, largest id], unknown ids mixed in: invalid UTF-8 is dense for ByteLevel"""
    t = tok(name)
    _, ent, pool = dc.images(dc.tokenizer_json(name))
    lossy = dc.CONFIGS[name][1]["type"] == "ByteLevel"
    rows = dc.random_rows(11, ent.size, 2000, 90)
    tk = helpers.wheel()
    ref = tk.Tokenizer.from_str(dc.tokenizer_json(name)) if tk else None
    for skip in (True, False):
        exp = ref.decode_batch(rows, skip_special_tokens=skip) if ref else [dc.table_decode(ent, pool, lossy, r, skip) for r in rows]
        got = all_paths(t, rows, skip)
        for path, g in got.items():
            assert g == exp, (name, path)


def test_edge_rows():
    t = tok("gpt2_bytelevel")
    v = t.get_vocab()
    sp, a = v["[SPEC]"], v["a"]
    assert t.decode_batch_csr(np.zeros(0, np.uint32), np.zeros(1, np.uint64))[1].tolist() == [0]
    assert t.decode_batch_rows(np.zeros((0, 4), np.int64)) == []
    rows = [[], [sp] * 40 + [a, v["the"]], [sp] * 33, [len(v) + 10, 0xFFFFFFFF, (1 << 20) - 1, a], [sp] * 31 + [v["b"]] + [a] * 40]
    exp_skip = ["", "a", "", "a", "b" + "a" * 40]   # ("the" is a special added token here)
    for got in all_paths(t, rows, True).values():
        assert got == exp_skip
    for got in all_paths(t, rows, False).values():
        assert got[1] == "[SPEC]" * 40 + "athe" and got[4].startswith("[SPEC]" * 31 + "b")


def _byte_ids(t):
    inv = {c: b for c, b in __import__("tokenizers_b200.tokenizer", fromlist=["_char_bytes"])._char_bytes().items()}
    v = t.get_vocab()
    return {b: v[c] for c, b in inv.items()}


def test_invalid_utf8_across_tokens_and_row_edges():
    t = tok("gpt2_bytelevel")
    bid = _byte_ids(t)
    raw = [b"\xe2\x82", b"\xac", b"\xe2\x82\xac", b"\xc0\xaf", b"\xe0\x80\xaf", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"\x80\xbf",
           b"a\xf0\x9f\x98", b"\x80b", b"\xf0\x9f\x98\x80", b"\xff\xfe", "€ok".encode()[:2] + b"x"]
    rows = [[bid[c] for c in r] for r in raw]
    exp = [r.decode("utf-8", "replace") for r in raw]
    for got in all_paths(t, rows, True).values():
        assert got == exp
    # split inside tokens: multi-byte tokens cut at every point into two rows and into one row of two tokens
    v = t.get_vocab()
    multi = [i for c, i in v.items() if len(dc.bytelevel_image(c)) >= 3][:200]
    rows = [[i] for i in multi] + [[multi[k], multi[k + 1]] for k in range(0, 198, 2)]
    ids, rp = csr(rows)
    got = texts(*t.decode_batch_csr(ids, rp))
    exp = [b"".join(dc.bytelevel_image(t.id_to_token(i)) for i in r).decode("utf-8", "replace") for r in rows]
    assert got == exp


def test_large_rows():
    t = tok("gpt2_bytelevel")
    _, ent, pool = dc.images(dc.tokenizer_json("gpt2_bytelevel"))
    rng = np.random.default_rng(3)
    one = rng.integers(0, 50257, size=10 ** 6)
    got = texts(*t.decode_batch_csr(one, np.array([0, one.size], np.uint64)))[0]
    assert got == dc.table_decode(ent, pool, True, one, True)
    lens = rng.integers(1, 4, size=10 ** 6)
    ids = rng.integers(0, 50257, size=int(lens.sum()))
    rp = np.zeros(lens.size + 1, np.uint64)
    np.cumsum(lens, out=rp[1:])
    text, off = t.decode_batch_csr(ids, rp)
    assert off.size == 10 ** 6 + 1
    sample = rng.integers(0, 10 ** 6, size=3000)
    for r in sample:
        row = ids[int(rp[r]):int(rp[r + 1])]
        assert text[int(off[r]):int(off[r + 1])].tobytes().decode("utf-8") == dc.table_decode(ent, pool, True, row, True)
    import torch
    a = np.zeros((10 ** 6, 3), np.int64)
    a[np.arange(3)[None, :] < lens[:, None]] = ids
    dev = t.decode_batch_rows(torch.from_numpy(a).cuda(), torch.from_numpy(lens).cuda())
    assert dev == texts(text, off)


def test_host_call_over_several_chunks(monkeypatch):
    monkeypatch.setenv("B2T_CHUNK_BYTES", "4096")   # 1024 ids per chunk
    t = Tokenizer.from_str(dc.tokenizer_json("wordpiece_cleanup"), device=0)
    g = GOLDEN["wordpiece_cleanup"]
    rows = g["rows"] * 10 + [list(np.random.default_rng(1).integers(0, 30522, 5000))] + g["rows"]
    exp = g["skip"] * 10 + [None] + g["skip"]
    ids, rp = csr(rows)
    got = texts(*t.decode_batch_csr(ids, rp))
    one = tok("wordpiece_cleanup").decode_batch_rows(np.array([rows[-len(g["rows"]) - 1]]))   # the long row, one chunk of its own
    assert got[len(g["rows"]) * 10] == one[0]
    assert [x for x, e in zip(got, exp) if e is not None] == [e for e in exp if e is not None]


def test_dense_rows_with_padding():
    tk = helpers.wheel()
    t = Tokenizer.from_str(dc.tokenizer_json("wordpiece_cleanup"), device=0)
    t.enable_padding(pad_id=0, length=64)
    t.enable_truncation(64)
    import corpus
    data, off = corpus.generate(4, 5, 0, 300)
    dn = t.encode_batch_dense(data, off, add_special_tokens=False)
    ids, ln = dn["input_ids"], dn["attention_mask"].sum(1).astype(np.int64)
    whole, cut = t.decode_batch_rows(ids), t.decode_batch_rows(ids, ln)
    if tk:
        ref = tk.Tokenizer.from_str(dc.tokenizer_json("wordpiece_cleanup"))
        assert whole == ref.decode_batch(ids.tolist()) and cut == ref.decode_batch([r[:n] for r, n in zip(ids.tolist(), ln.tolist())])
    import torch
    assert t.decode_batch_rows(torch.from_numpy(ids.astype(np.int64)).cuda(), torch.from_numpy(ln).cuda()) == cut


@pytest.mark.parametrize("asset", ["gpt2_style", "llama3_style"])
def test_round_trip_of_the_corpus(asset):
    """device encode, then device decode: byte-level BPE gives the input bytes back (the corpus is valid UTF-8)"""
    import torch, corpus
    j = json.loads(helpers.asset_json(asset)); j["decoder"] = dc.BYTELEVEL
    t = Tokenizer.from_str(json.dumps(j), device=0)
    data, off = corpus.generate(2, 21, 0, 20000)
    reps = max(1, (50 << 20) // len(data))   # a tiled batch of about 50 MiB
    big = np.tile(data, reps)
    boff = np.concatenate([off[:-1] + k * len(data) for k in range(reps)] + [np.array([reps * len(data)], np.uint64)]).astype(np.uint64)
    be = t.encode_batch_csr(big, boff, offsets=False, word_ids=False)
    text, toff = t.decode_batch_csr(be.ids, be.row_ptr)
    assert np.array_equal(toff, boff) and np.array_equal(text, big)
    L = _lib.lib()
    d_ids = torch.from_numpy(be.ids.astype(np.int64)).cuda().to(torch.int32)
    d_rp = torch.from_numpy(be.row_ptr.astype(np.int64)).cuda()
    import ctypes
    res = ctypes.c_void_p()
    _lib.check(L.b2t_decode_batch_device(t.handle, d_ids.data_ptr(), d_ids.numel(), d_rp.data_ptr(), None, boff.size - 1, 1,
                                         torch.cuda.current_stream().cuda_stream, ctypes.byref(res)))
    assert L.b2t_result_on_device(res) == 1 and L.b2t_result_n_tokens(res) == big.size
    from tokenizers_b200.tokenizer import _device_view
    dt = _device_view(torch, L.b2t_result_text(res), big.size, torch.uint8, d_ids.device)
    assert torch.equal(dt, torch.from_numpy(big).cuda())
    L.b2t_result_free(res)


def test_concurrent_host_decodes_and_encodes():
    t = tok("gpt2_bytelevel")
    g = GOLDEN["gpt2_bytelevel"]
    ids, rp = csr(g["rows"])
    import corpus
    data, off = corpus.generate(2, 4, 0, 3000)
    enc = t.encode_batch_csr(data, off)
    errors = []

    def work(k):
        try:
            for _ in range(5):
                if k % 2:
                    assert texts(*t.decode_batch_csr(ids, rp)) == g["skip"]
                else:
                    assert np.array_equal(t.encode_batch_csr(data, off).ids, enc.ids)
        except Exception as ex:   # (reported below)
            errors.append(ex)
    th = [threading.Thread(target=work, args=(k,)) for k in range(6)]
    [x.start() for x in th]
    [x.join() for x in th]
    assert not errors, errors


def test_add_tokens_changes_decode():
    t = Tokenizer.from_str(dc.tokenizer_json("wordpiece_cleanup"), device=0)
    n = t.get_vocab_size()
    assert t.decode_batch_rows(np.array([[n, 5]])) == [t.decode([n, 5])]
    t.add_tokens(["brandnew"])
    t.add_special_tokens(["<late>"])
    assert t.decode_batch_rows(np.array([[n, n + 1, 5]]), skip_special_tokens=True) == [t.decode([n, n + 1, 5])]
    assert t.decode_batch_rows(np.array([[n, n + 1]]), skip_special_tokens=False) == ["brandnew <late>"]


def test_error_paths():
    import torch
    j = json.loads(helpers.asset_json("wordpiece")); j["decoder"] = {"type": "Metaspace", "replacement": "▁"}
    t = Tokenizer.from_str(json.dumps(j), device=0)   # construction succeeds, encode works
    assert t.encode_batch_csr(*helpers.pack_docs(["hello world"])).ids.size > 0
    with pytest.raises(UnsupportedConfig, match="Metaspace"):
        t.decode_batch_rows(np.array([[1, 2]]))
    with pytest.raises(UnsupportedConfig):
        t.decode_batch_csr(np.array([1]), np.array([0, 1]))
    t = tok("wordpiece_cleanup")
    with pytest.raises(B2TError) as ei:
        t.decode_batch_csr(np.array([1, 2, 3]), np.array([0, 2, 1, 3]))
    assert ei.value.code == _lib.B2T_ERR_INVALID
    with pytest.raises(B2TError) as ei:
        t.decode_batch_csr(np.array([1, 2, 3]), np.array([0, 4]))
    assert ei.value.code == _lib.B2T_ERR_INVALID
    for bad in (np.array([[1, -1]]), np.array([[1, 1 << 32]]), torch.tensor([[1, -3]]).cuda(), torch.tensor([[1 << 33, 1]]).cuda()):
        with pytest.raises(ValueError):
            t.decode_batch_rows(bad)
    L = _lib.lib()
    import ctypes
    res = ctypes.c_void_p()
    ids = torch.tensor([1, 2, 3], dtype=torch.int32).cuda()
    rp = torch.tensor([0, 2, 1, 3], dtype=torch.int64).cuda()
    assert L.b2t_decode_batch_device(t.handle, ids.data_ptr(), 3, rp.data_ptr(), None, 3, 0, None, ctypes.byref(res)) == _lib.B2T_ERR_INVALID
    rp = torch.tensor([0, 5], dtype=torch.int64).cuda()
    assert L.b2t_decode_batch_device(t.handle, ids.data_ptr(), 3, rp.data_ptr(), None, 1, 0, None, ctypes.byref(res)) == _lib.B2T_ERR_INVALID
    assert L.b2t_decode_batch(t.handle, None, 3, None, None, 1, 0, ctypes.byref(res)) == _lib.B2T_ERR_INVALID
    assert L.b2t_engine_set_decoder(t.handle, None) == 0   # no decoder now
    assert L.b2t_decode_batch(t.handle, np.array([1], np.uint32).ctypes.data, 1, np.array([0, 1], np.uint64).ctypes.data, None, 1, 0,
                              ctypes.byref(res)) == _lib.B2T_ERR_INVALID
    assert "no decoder" in L.b2t_last_error().decode()
    t._set_decoder()
    assert t.decode_batch_rows(np.array([[5]])) == [t.decode([5])]


def test_encode_results_have_no_text_views():
    t = tok("gpt2_bytelevel")
    L = _lib.lib()
    import ctypes
    data, off = helpers.pack_docs(["hello world"] * 3)
    g = GOLDEN["gpt2_bytelevel"]
    t.decode_batch_csr(*csr(g["rows"]))   # a pooled result that held text
    res = ctypes.c_void_p()
    _lib.check(L.b2t_encode_batch(t.handle, data.ctypes.data, off.ctypes.data, 3, 0, ctypes.byref(res)))
    assert not L.b2t_result_text(res) and not L.b2t_result_text_off(res)
    L.b2t_result_free(res)


def test_long_images_and_every_row_alignment():
    """D2's window: steps whose images exceed it (tokens of up to 512 bytes), stored lane by lane, between steps stored in
    16-byte blocks; rows that start at every offset of a block and end inside one"""
    name = "vocabgen_bpe_high"
    t = tok(name)
    _, ent, pool = dc.images(dc.tokenizer_json(name))
    ex = [i for i in range(ent.size) if dc.entry(ent, pool, i)[0]]
    by_len = sorted(ex, key=lambda i: len(dc.entry(ent, pool, i)[2]))
    short, long = by_len[:200], by_len[-40:]
    assert len(dc.entry(ent, pool, long[-1])[2]) >= 256
    rng = np.random.default_rng(9)
    rows = []
    for k in range(600):
        n = int(rng.integers(0, 120))
        mix = long if k % 3 == 0 else short
        rows.append([int(rng.choice(mix)) if rng.random() < 0.7 else int(rng.choice(short)) for _ in range(n)])
        rows.append([int(rng.choice(short))] * (k % 17))   # (moves the next row's start through every block offset)
    for skip in (True, False):
        exp = [dc.table_decode(ent, pool, True, r, skip) for r in rows]
        for path, got in all_paths(t, rows, skip).items():
            assert got == exp, path
