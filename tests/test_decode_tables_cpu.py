"""CPU: the decoder table the device decode kernels read (b2t_decoder_images) against the reference wheel, its refusals, and
the kernels' lossy UTF-8 classifier (compiled for the host by tests/native/decode_emul.cpp) against Python's
bytes.decode("utf-8", "replace"), which equals the reference's String::from_utf8_lossy."""
import ctypes, itertools, json, os, random
import numpy as np
import pytest
import helpers
import decode_cases as dc
from tokenizers_b200 import _lib

EDGE_BYTES = [0x00, 0x41, 0x7F, 0x80, 0x8F, 0x90, 0x9F, 0xA0, 0xBF, 0xC0, 0xC1, 0xC2, 0xDF, 0xE0, 0xE1, 0xEC, 0xED, 0xEE, 0xEF,
              0xF0, 0xF1, 0xF3, 0xF4, 0xF5, 0xFF]


# ---------------------------------------------------------------------------------------------- the lossy classifier
def _emul():
    path = os.path.join(helpers.ROOT, "tests", "native", "libdecode_emul.so")
    if not os.path.exists(path):
        pytest.skip("tests/native/libdecode_emul.so is not built (__graft_entry__.build())")
    L = ctypes.CDLL(path)
    L.b2t_emul_lossy.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_uint32] + [ctypes.c_void_p] * 2
    L.b2t_emul_lossy.restype = ctypes.c_uint64
    return L


def _check_rows(rows):
    """every row through the classifier on its own == bytes.decode("utf-8", "replace") of the row"""
    L = _emul()
    data = np.frombuffer(b"".join(rows), dtype=np.uint8).copy()
    off = np.zeros(len(rows) + 1, dtype=np.uint64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    out, out_off = np.zeros(3 * data.size + 16, np.uint8), np.zeros(len(rows) + 1, np.uint64)
    n = L.b2t_emul_lossy(data.ctypes.data, off.ctypes.data, len(rows), out.ctypes.data, out_off.ctypes.data)
    assert n != 2 ** 64 - 1, "a row's count and its rewrite disagree"
    got = out[:n].tobytes()
    # an ASCII byte ends every invalid subpart and is valid itself: decoding rows joined by "\n" decodes each row alone
    exp = b"\n".join(rows).decode("utf-8", "replace").encode("utf-8")
    o = out_off.tolist()
    if b"\n".join(got[o[i]:o[i + 1]] for i in range(len(rows))) != exp:
        for i, r in enumerate(rows):
            assert got[o[i]:o[i + 1]] == r.decode("utf-8", "replace").encode("utf-8"), r.hex()


def test_lossy_classifier_every_short_string():
    rows = [bytes(p) for n in (1, 2) for p in itertools.product(range(256), repeat=n)]
    _check_rows(rows)


def test_lossy_classifier_utf8_range_edges():
    for n in range(1, 6):
        _check_rows([bytes(p) for p in itertools.product(EDGE_BYTES, repeat=n)])


def test_lossy_classifier_random_and_row_edges():
    rng = random.Random(7)
    hi = list(range(0x80, 0x100)) + [0x41, 0x20]
    rows = [bytes(rng.choice(hi) for _ in range(rng.randint(3, 40))) for _ in range(100000)]
    rows += ["€ ü 𝒷 ok".encode()[:k] for k in range(13)] + [b"\xe2\x82", b"\xac", b"\xf0\x9f", b"\x98\x80", b"\xed\xa0\x80", b"\xf4\x90\x80\x80",
                                                           b"\xc0\xaf", b"\xe0\x80\xaf", b"\xbf\xbf\xbf\xbf"]
    _check_rows(rows)


# ---------------------------------------------------------------------------------------------- the decoder table
def _wheel_or_skip():
    tk = helpers.wheel()
    if tk is None:
        pytest.skip("reference wheel not importable")
    return tk


@pytest.mark.parametrize("name", list(dc.CONFIGS))
def test_decoder_images_match_the_wheel(name):
    tk = _wheel_or_skip()
    tj = dc.tokenizer_json(name)
    rc, ent, pool = dc.images(tj)
    assert rc == 0
    ref = tk.Tokenizer.from_str(tj)
    kind = dc.CONFIGS[name][1]
    lossy = kind is not None and kind["type"] == "ByteLevel"
    vocab = ref.get_vocab(with_added_tokens=True)
    a = vocab["a"]
    n = ent.size
    assert n == max(vocab.values()) + 1
    # (ids up to 2^20 - 1: every id of the vocabulary's top 20 000, a random sample of the rest and the added tokens)
    ids = list(range(n)) if n <= 200000 else sorted(set(random.Random(1).sample(range(n), 20000)) | set(range(n - 20000, n)) |
                                                    {vocab[c] for c, _ in dc.ADDED})
    special = {t.content for t in ref.get_added_tokens_decoder().values() if t.special}
    first = ref.decode_batch([[i] for i in ids], skip_special_tokens=False)
    pair = ref.decode_batch([[a, i] for i in ids], skip_special_tokens=False)
    head = ref.decode([a], skip_special_tokens=False)
    checked = existing = 0
    for i, f, p in zip(ids, first, pair):
        ex, sk, img1, img2 = dc.entry(ent, pool, i)
        tok = ref.id_to_token(i)
        assert ex == (tok is not None), i
        if not ex:
            continue
        existing += 1
        assert sk == (tok in special), i
        if lossy:
            assert img1 == img2 == dc.bytelevel_image(tok), i
            try:
                img1.decode("utf-8")
            except UnicodeDecodeError:
                continue
        assert img1.decode("utf-8") == f, (i, tok)
        assert p.startswith(head) and img2.decode("utf-8") == p[len(head):], (i, tok)
        checked += 1
    assert checked > existing // 2


@pytest.mark.parametrize("name", ["gpt2_bytelevel", "wordpiece_cleanup", "wordpiece_no_decoder", "vocabgen_wordpiece_high"])
def test_table_restatement_decodes_like_the_wheel(name):
    """decode() restated over the table == the wheel's decode_batch on random rows (invalid UTF-8 is dense for ByteLevel)"""
    tk = _wheel_or_skip()
    tj = dc.tokenizer_json(name)
    _, ent, pool = dc.images(tj)
    ref = tk.Tokenizer.from_str(tj)
    lossy = dc.CONFIGS[name][1] is not None and dc.CONFIGS[name][1]["type"] == "ByteLevel"
    vocab = ref.get_vocab(with_added_tokens=True)
    rows = dc.random_rows(3, ent.size, 400, 40, extra=[vocab[c] for c, _ in dc.ADDED])
    rows += [[vocab["[SPEC]"]] * 40 + [vocab["a"]], [vocab["the"], vocab["a"], vocab["do not"], vocab["' x"]], []]
    for skip in (True, False):
        exp = ref.decode_batch([[min(i, 0xFFFFFFFF) for i in r] for r in rows], skip_special_tokens=skip)
        assert [dc.table_decode(ent, pool, lossy, r, skip) for r in rows] == exp


def test_cleanup_runs_on_each_token_alone():
    tk = _wheel_or_skip()
    tj = dc.tokenizer_json("wordpiece_cleanup")
    _, ent, pool = dc.images(tj)
    ref = tk.Tokenizer.from_str(tj)
    v = ref.get_vocab()
    for row in ([v["c"], v["' x"]], [v["[SPEC]"], v["a"]], [v["a"], v["do not"], v["b"]]):
        for skip in (True, False):
            assert dc.table_decode(ent, pool, False, row, skip) == ref.decode(row, skip_special_tokens=skip)


def test_refusals():
    tj = dc.tokenizer_json("wordpiece_cleanup")
    for dec in ({"type": "Sequence", "decoders": []}, {"type": "Metaspace"}, {"type": "ByteFallback"}):
        rc, _, _ = dc.images(tj, decoder=dec)
        assert rc == _lib.B2T_ERR_UNSUPPORTED
    # an unknown kind reaching the C ABI
    from tokenizers_b200.tokenizer import parse_tokenizer_json, engine_config, decoder_spec
    cfg = parse_tokenizer_json(json.loads(tj))
    c, keep = engine_config(cfg)
    sp, keep2 = decoder_spec(None, [])
    sp.kind = 7
    n, nb = ctypes.c_uint32(), ctypes.c_uint64()
    assert _lib.lib().b2t_decoder_images(ctypes.byref(c), ctypes.byref(sp), None, None, ctypes.byref(n), ctypes.byref(nb)) == _lib.B2T_ERR_UNSUPPORTED
    # normalized=true added tokens behind a BertNormalizer: refused; without the normalizer, or when not normalized, accepted
    norm = _lib.NORM_BERT | _lib.NORM_LOWERCASE
    added = [dc.SimpleNamespace(content="HeLLo Wörld", id=40000, special=False, normalized=True)]
    assert dc.images(tj, normalizer_flags=norm, added=added)[0] == _lib.B2T_ERR_UNSUPPORTED
    assert "normalized" in _lib.lib().b2t_last_error().decode()
    assert dc.images(tj, normalizer_flags=0, added=added)[0] == 0
    added[0].normalized = False
    assert dc.images(tj, normalizer_flags=norm, added=added)[0] == 0


def test_refused_decoder_does_not_fail_parsing():
    """parse_tokenizer_json keeps an unsupported decoder: only device decode is unavailable"""
    from tokenizers_b200.tokenizer import parse_tokenizer_json, decoder_spec
    j = json.loads(helpers.asset_json("gpt2_style"))
    j["decoder"] = {"type": "Sequence", "decoders": [{"type": "ByteFallback"}]}
    cfg = parse_tokenizer_json(j)
    sp, reason = decoder_spec(cfg["decoder"], [])
    assert sp is None and "Sequence" in reason
