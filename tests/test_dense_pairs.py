"""Dense mode for pairs of sequences (b2t_encode_pairs_dense*): pair truncation, the pair template with type ids, padding.
CPU: the plain restatement (pair_oracle.dense_pair_rows) against the reference wheel and the committed fixture, the pair
kernels' own truncation algebra (dense_kernels.cuh pair_keep, compiled for the host by tests/native/dense_emul.cpp) against
the restatement on every small input, and the spec the shim builds.  GPU: the engine against all of them."""
import ctypes, gzip, json, os, subprocess
import numpy as np
import pytest
import helpers, fuzzgen, corpus
import pair_oracle as po
from oracle import oracle as orc

tk = helpers.wheel()
HERE = os.path.dirname(os.path.abspath(__file__))
STRATEGIES = ("longest_first", "only_first", "only_second")
TOO_SHORT = "Truncation error: Sequence to truncate too short to respect the provided max_length"


def _template_b_first(v):
    """TemplateProcessing with B before A, a special token of two ids and type ids 0 / 1 / 2"""
    return {"type": "TemplateProcessing",
            "single": [{"SpecialToken": {"id": "[CLS]", "type_id": 2}}, {"Sequence": {"id": "A", "type_id": 0}}],
            "pair": [{"SpecialToken": {"id": "[CLS]", "type_id": 2}}, {"Sequence": {"id": "B", "type_id": 1}},
                     {"SpecialToken": {"id": "<two>", "type_id": 0}}, {"Sequence": {"id": "A", "type_id": 0}},
                     {"SpecialToken": {"id": "[CLS]", "type_id": 2}}],
            "special_tokens": {"[CLS]": {"id": "[CLS]", "ids": [v["[CLS]"]], "tokens": ["[CLS]"]},
                               "<two>": {"id": "<two>", "ids": [v["[SEP]"], v["[MASK]"]], "tokens": ["[SEP]", "[MASK]"]}}}


# name -> (asset, post-processor from the vocabulary)
TEMPLATES = {
    "bert": ("wordpiece", lambda v: {"type": "BertProcessing", "sep": ["[SEP]", v["[SEP]"]], "cls": ["[CLS]", v["[CLS]"]]}),
    "roberta": ("gpt2_style", lambda v: {"type": "RobertaProcessing", "sep": ["b", v["b"]], "cls": ["a", v["a"]],
                                         "trim_offsets": True, "add_prefix_space": False}),
    "b_first": ("wordpiece", _template_b_first),
    "none": ("llama3_style", lambda v: None),
}
# (truncation | None, padding); max_length "special" = exactly the special tokens of the template: a budget of 0
SETTINGS = [
    (dict(max_length=40, strategy="longest_first", direction="right"), dict(length=40, direction="right", pad_id=0, pad_type_id=0)),
    (dict(max_length=33, strategy="longest_first", direction="left"), dict(length=None, direction="left", pad_id=3, pad_type_id=1)),
    (dict(max_length=30, strategy="only_first", direction="right"), dict(length=None, direction="right", pad_id=1, pad_type_id=2, pad_to_multiple_of=8)),
    (dict(max_length=24, strategy="only_second", direction="left"), dict(length=40, direction="left", pad_id=5, pad_type_id=0, pad_to_multiple_of=16)),
    (dict(max_length=40, strategy="only_first", direction="left"), dict(length=None, direction="right", pad_id=2, pad_type_id=7)),
    (dict(max_length=36, strategy="only_second", direction="right"), dict(length=None, direction="left", pad_id=2, pad_type_id=0)),
    (None, dict(length=None, direction="right", pad_id=2, pad_type_id=0)),
    (dict(max_length="special", strategy="only_first", direction="right"), dict(length=None, direction="right", pad_id=9, pad_type_id=3)),
]


def tokenizer_json(name):
    asset, pp = TEMPLATES[name]
    js = json.loads(helpers.asset_json(asset))
    js["post_processor"] = pp(js["model"]["vocab"])
    return json.dumps(js)


WORDS = ["the", "cat", "sat", "on", "a", "mat", "why", "not", "blue", "run"]


def pairs_for(seed, n=150):
    """(fuzz document, short sentence of at most four words) pairs, and the empty corner cases"""
    import random
    rng = random.Random(seed)
    long_ = fuzzgen.rand_docs(seed, n, max_len=90)
    short = [" ".join(rng.choice(WORDS) for _ in range(rng.randint(0, 4))) for _ in range(n)]
    return list(zip(long_, short)) + [("", ""), ("a", ""), ("", "b"), ("hello world " * 8, "x")]


def arrange(pairs, tr):
    """the pairs a setting runs on: the short sentence second for only_first and first for only_second (so that the
    strategy's sequence can always be cut), alternating otherwise (so that longest_first sees both orders)"""
    if tr is not None and tr["strategy"] == "only_first":
        return pairs
    if tr is not None and tr["strategy"] == "only_second":
        return [(b, a) for a, b in pairs]
    return [(a, b) if k % 2 else (b, a) for k, (a, b) in enumerate(pairs)]


def n_special(js):
    from tokenizers_b200.tokenizer import parse_post_processor, special_token_count
    return special_token_count(parse_post_processor(json.loads(js).get("post_processor")), True)


def resolve(js, tr):
    """the setting's truncation with max_length "special" resolved; None where it has no dense form (max_length 0)"""
    if tr is None or tr["max_length"] != "special":
        return tr
    m = n_special(js)
    return dict(tr, max_length=m) if m else None


def pieces_of(js, add_special_tokens):
    from tokenizers_b200.tokenizer import parse_post_processor
    tp = parse_post_processor(json.loads(js).get("post_processor"))
    pieces = [("seq", 0, 0), ("seq", 1, 1)] if tp is None else tp["pair"]
    return [p for p in pieces if p[0] == "seq" or add_special_tokens]


def oracle_rows(ids, rp, js, tr, pd, add_special_tokens):
    """pair_oracle.dense_pair_rows with the settings -> (ids, type ids, mask, lengths) or the error message"""
    try:
        return po.dense_pair_rows(ids, rp, length=pd["length"] or 0, pad_to_multiple_of=pd.get("pad_to_multiple_of") or 0,
                                  max_length=tr["max_length"] if tr else 0, strategy=tr["strategy"] if tr else "longest_first",
                                  truncate_left=bool(tr and tr["direction"] == "left"), pad_id=pd["pad_id"], pad_type_id=pd["pad_type_id"],
                                  pad_left=pd["direction"] == "left", pieces=pieces_of(js, add_special_tokens))
    except ValueError as ex:
        return str(ex)


def wheel_rows(js, pairs, tr, pd, add_special_tokens):
    """the reference: encode_batch on the pairs with truncation and padding, the Encodings stacked"""
    tok = tk.Tokenizer.from_str(js)
    if tr:
        tok.enable_truncation(tr["max_length"], strategy=tr["strategy"], direction=tr["direction"])
    tok.enable_padding(direction=pd["direction"], pad_id=pd["pad_id"], pad_type_id=pd["pad_type_id"], length=pd["length"],
                       pad_to_multiple_of=pd.get("pad_to_multiple_of"))
    try:
        encs = tok.encode_batch(pairs, add_special_tokens=add_special_tokens)
    except Exception as ex:
        return str(ex)
    n = len(pairs)
    return (np.array([e.ids for e in encs], dtype=np.uint32).reshape(n, -1), np.array([e.type_ids for e in encs], dtype=np.uint8).reshape(n, -1),
            np.array([e.attention_mask for e in encs], dtype=np.uint8).reshape(n, -1),
            np.array([sum(e.attention_mask) for e in encs], dtype=np.uint32))


def oracle_csr(js, pairs):
    ids, _, _, rp = orc.Oracle(js).encode_batch([s for p in pairs for s in p])
    return ids, rp


def same(got, exp, what):
    """(ids, type ids, mask, lengths) or an error message, both sides"""
    if isinstance(exp, str) or isinstance(got, str):
        assert isinstance(exp, str) and isinstance(got, str) and TOO_SHORT in exp and TOO_SHORT in got, (what, got if isinstance(got, str) else "rows", exp if isinstance(exp, str) else "rows")
        return
    for g, e, nm in zip(got, exp, ("ids", "type_ids", "mask", "lengths")):
        assert g.shape == e.shape and np.array_equal(g, e), (what, nm, g.shape, e.shape)


def cases():
    for k, (tr, pd) in enumerate(SETTINGS):
        for ast in (True, False):
            yield f"{k}/{int(ast)}", tr, pd, ast


def _golden():
    return json.loads(gzip.open(os.path.join(helpers.GOLDEN, "golden_dense_pairs.json.gz")).read().decode("utf-8"))


def golden_rows(c):
    if "error" in c:
        return c["error"]
    shape = tuple(c["shape"])
    return (np.array(c["ids"], dtype=np.uint32).reshape(shape), np.array(c["type_ids"], dtype=np.uint8).reshape(shape),
            np.array(c["mask"], dtype=np.uint8).reshape(shape), np.array(c["lengths"], dtype=np.uint32))


# ------------------------------------------------------------------------------------------------------------- CPU
def test_settings_reach_their_cases():
    """the settings cut with every strategy, hit budget 0 and the SequenceTooShort error on the test pairs"""
    js = tokenizer_json("bert")
    for tr, _ in SETTINGS:
        tr = resolve(js, tr)
        if tr is None:
            continue
        ids, rp = oracle_csr(js, arrange(pairs_for(11), tr))
        lens = np.diff(rp.astype(np.int64)).reshape(-1, 2)
        budget = tr["max_length"] - n_special(js)
        kept = [po.pair_keep(int(a), int(b), budget, tr["strategy"]) for a, b in lens]
        assert all(k is not None for k in kept) and any(k != (a, b) for k, (a, b) in zip(kept, lens.tolist())), tr
    assert po.pair_keep(6, 2, 1, "only_first") is None and po.pair_keep(6, 0, 0, "only_first") == (0, 0)


def _emul():
    so = os.path.join(HERE, "native", "libdense_emul.so")
    src = os.path.join(HERE, "native", "dense_emul.cpp")
    hdr = os.path.join(helpers.ROOT, "tokenizers_b200", "csrc", "dense_kernels.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        inc = "/usr/local/cuda/include"
        if not os.path.exists(os.path.join(inc, "cuda_runtime.h")):
            pytest.skip("CUDA headers not available")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + inc, "-Wno-attributes", "-shared", "-fPIC", "-o", so, src])
    L = ctypes.CDLL(so)
    L.b2t_emul_pair_keep.restype = None
    L.b2t_emul_pair_keep.argtypes = [ctypes.c_uint32] + [ctypes.c_void_p] * 7
    return L


def test_pair_keep_kernel_algebra_exhaustive():
    """dense_kernels.cuh pair_keep == the restatement for every n1, n2, budget in [0, 48] and every strategy (which inputs
    fail included), and with no truncation at all"""
    L = _emul()
    r = np.arange(49, dtype=np.uint32)
    n1, n2, bud = (a.reshape(-1) for a in np.meshgrid(r, r, np.append(r, np.uint32(0xFFFFFFFF)), indexing="ij"))
    for s, name in enumerate(STRATEGIES):
        st = np.full(n1.size, s, dtype=np.uint32)
        k1, k2, ok = np.zeros_like(n1), np.zeros_like(n1), np.zeros(n1.size, dtype=np.uint8)
        L.b2t_emul_pair_keep(n1.size, n1.ctypes.data, n2.ctypes.data, bud.ctypes.data, st.ctypes.data, k1.ctypes.data, k2.ctypes.data, ok.ctypes.data)
        for i in range(n1.size):
            b = int(bud[i])
            exp = po.pair_keep(int(n1[i]), int(n2[i]), None if b == 0xFFFFFFFF else b, name)
            got = (int(k1[i]), int(k2[i])) if ok[i] else None
            assert got == exp, (name, int(n1[i]), int(n2[i]), b, got, exp)
        assert not ok.all() or s == 0   # the only_* strategies do fail on some inputs


@pytest.mark.skipif(tk is None, reason="reference wheel not importable")
@pytest.mark.parametrize("name", list(TEMPLATES))
def test_dense_pair_rows_matches_wheel(name):
    js = tokenizer_json(name)
    for key, tr, pd, ast in cases():
        tr = resolve(js, tr)
        pairs = arrange(pairs_for(11), tr)
        same(oracle_rows(*oracle_csr(js, pairs), js, tr, pd, ast), wheel_rows(js, pairs, tr, pd, ast), (name, key))


@pytest.mark.parametrize("name", list(TEMPLATES))
def test_dense_pair_rows_matches_golden(name):
    """the same restatement against committed vectors of the wheel (no wheel needed)"""
    g = _golden()
    js = tokenizer_json(name)
    for key, tr, pd, ast in cases():
        c = g["cases"].get(f"{name}/{key}")
        tr = resolve(js, tr)
        if c is None:
            assert tr is None
            continue
        pairs = arrange([tuple(p) for p in g["pairs"]], tr)
        same(oracle_rows(*oracle_csr(js, pairs), js, tr, pd, ast), golden_rows(c), (name, key))
    for k, (a, b, tr) in enumerate(ERROR_CASES):
        same(oracle_rows(*oracle_csr(js, [(a, b)]), js, tr, SETTINGS[0][1], True), golden_rows(g["cases"][f"{name}/error{k}"]), (name, k))


# pairs with a cut the strategy cannot make: SequenceTooShort (B alone fills the budget / A alone does / A would go to 0)
ERROR_CASES = [
    ("hello", "the second sequence is much longer than this budget " * 2, dict(max_length=16, strategy="only_first", direction="right")),
    ("the first sequence is much longer than this budget " * 2, "hi", dict(max_length=16, strategy="only_second", direction="left")),
]


def _apply(tok, tr, pd):
    tok.no_truncation(); tok.no_padding()
    if tr:
        tok.enable_truncation(tr["max_length"], stride=tr.get("stride", 0), strategy=tr["strategy"], direction=tr["direction"])
    tok.enable_padding(direction=pd["direction"], pad_id=pd["pad_id"], pad_type_id=pd["pad_type_id"], length=pd["length"],
                       pad_to_multiple_of=pd.get("pad_to_multiple_of"))


def spec_rows(tok, ids, rp, add_special_tokens):
    """the b2t_pair_dense_spec the shim builds, fed to the restatement"""
    sp, keep = tok.pair_dense_spec(add_special_tokens)
    from tokenizers_b200 import _lib
    pids, ptypes = keep
    pieces = [("seq", 0 if i == _lib.PIECE_A else 1, int(t)) if i in (_lib.PIECE_A, _lib.PIECE_B) else ("special", int(i), int(t))
              for i, t in zip(pids.tolist(), ptypes.tolist())]
    assert sp.n_pieces == len(pieces) and sp.struct_size == ctypes.sizeof(_lib.PairDenseSpec)
    try:
        return po.dense_pair_rows(ids, rp, length=sp.length, pad_to_multiple_of=sp.pad_to_multiple_of, max_length=sp.max_length,
                                  strategy=STRATEGIES[sp.strategy], truncate_left=bool(sp.truncate_left), pad_id=sp.pad_id,
                                  pad_type_id=sp.pad_type_id, pad_left=bool(sp.pad_left), pieces=pieces)
    except ValueError as ex:
        return str(ex)


@pytest.mark.parametrize("name", list(TEMPLATES))
def test_pair_dense_spec_matches_wheel(name):
    """Tokenizer.pair_dense_spec (the shim's settings -> b2t_pair_dense_spec), read back into the restatement, gives the
    reference's rows: the committed vectors always, the wheel when it is importable"""
    js = tokenizer_json(name)
    tok = helpers.oracle_backed_tokenizer(js)
    g = _golden()
    for key, tr, pd, ast in cases():
        tr = resolve(js, tr)
        if tr is None and SETTINGS[int(key.split("/")[0])][0] is not None:
            continue
        _apply(tok, tr, pd)
        gpairs = arrange([tuple(p) for p in g["pairs"]], tr)
        same(spec_rows(tok, *oracle_csr(js, gpairs), ast), golden_rows(g["cases"][f"{name}/{key}"]), (name, key, "golden"))
        if tk is not None:
            pairs = arrange(pairs_for(11), tr)
            same(spec_rows(tok, *oracle_csr(js, pairs), ast), wheel_rows(js, pairs, tr, pd, ast), (name, key, "wheel"))


def test_pair_dense_spec_refusals():
    from tokenizers_b200 import UnsupportedConfig
    js = json.loads(tokenizer_json("b_first"))
    tok = helpers.oracle_backed_tokenizer(json.dumps(js))
    _apply(tok, dict(max_length=32, strategy="longest_first", direction="right", stride=4), SETTINGS[0][1])
    with pytest.raises(UnsupportedConfig):   # overflowing parts have no dense form
        tok.pair_dense_spec()
    _apply(tok, dict(max_length=3, strategy="longest_first", direction="right"), SETTINGS[0][1])
    with pytest.raises(ValueError):          # max_length below the 5 special tokens of the pair template
        tok.pair_dense_spec()
    tok.no_padding()
    with pytest.raises(UnsupportedConfig):
        tok.pair_dense_spec()
    js["post_processor"]["pair"] = []          # a template without a pair form
    tok = helpers.oracle_backed_tokenizer(json.dumps(js))
    _apply(tok, None, SETTINGS[0][1])
    with pytest.raises(ValueError, match="no template for pairs"):
        tok.pair_dense_spec()


# ------------------------------------------------------------------------------------------------------------- GPU
def engine_rows(tok, pairs, tr, pd, add_special_tokens=True):
    _apply(tok, tr, pd)
    try:
        out = tok.encode_pairs_dense(pairs, add_special_tokens=add_special_tokens)
    except ValueError as ex:
        if TOO_SHORT not in str(ex):
            raise
        return str(ex)
    return out["input_ids"], out["token_type_ids"], out["attention_mask"], out["lengths"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TEMPLATES))
def test_gpu_pairs_match_oracle_wheel_and_golden(name):
    from tokenizers_b200 import Tokenizer
    js = tokenizer_json(name)
    tok = Tokenizer.from_str(js)
    g = _golden()
    for key, tr, pd, ast in cases():
        tr0, tr = tr, resolve(js, tr)
        if tr is None and tr0 is not None:
            continue
        pairs, gpairs = arrange(pairs_for(12), tr), arrange([tuple(p) for p in g["pairs"]], tr)
        got = engine_rows(tok, pairs, tr, pd, ast)
        same(got, oracle_rows(*oracle_csr(js, pairs), js, tr, pd, ast), (name, key, "oracle"))
        if tk is not None:
            same(got, wheel_rows(js, pairs, tr, pd, ast), (name, key, "wheel"))
        same(engine_rows(tok, gpairs, tr, pd, ast), golden_rows(g["cases"][f"{name}/{key}"]), (name, key, "golden"))
    for k, (a, b, tr) in enumerate(ERROR_CASES):   # SequenceTooShort: the whole batch fails with the reference's message
        _apply(tok, tr, SETTINGS[0][1])
        with pytest.raises(ValueError, match="too short"):
            tok.encode_pairs_dense(pairs_for(12)[:5] + [(a, b)])


def chunk_pairs():
    """consecutive corpus documents paired up, pairs whose A ends just before or just after a 64 KiB boundary of the batch
    (a byte-based cut would fall between A and B), and one pair larger than a chunk"""
    data, off = corpus.generate(2, 31, 0, 3000)
    docs = corpus.to_strings(data, off)
    pairs = list(zip(docs[0::2], docs[1::2]))
    filler = "lorem ipsum dolor sit amet, consectetur adipiscing elit "
    pos = sum(len(a.encode()) + len(b.encode()) for a, b in pairs)
    for delta in (-3, 0, 5):
        gap = (-pos) % 65536 + delta + 65536
        a = (filler * (gap // len(filler) + 1))[:gap]
        pairs.append((a, "the second sequence starts on the other side"))
        pos += len(a.encode()) + len(pairs[-1][1].encode())
    pairs.append(((filler * 800)[:40000], (filler * 800)[:40000]))   # 80 000 bytes: more than one chunk
    return pairs + list(zip(docs[1::2], docs[2::2]))[:200]


@pytest.mark.gpu
def test_gpu_pairs_multi_chunk_batch_longest_and_device_entry(monkeypatch):
    from tokenizers_b200 import Tokenizer, _lib
    import torch
    js = tokenizer_json("roberta")
    pairs = chunk_pairs()
    ids, rp = oracle_csr(js, pairs)
    tr, pd = dict(max_length=64, strategy="longest_first", direction="right"), dict(length=64, direction="right", pad_id=9, pad_type_id=1)
    tr2, pd2 = dict(max_length=100, strategy="longest_first", direction="left"), dict(length=None, direction="left", pad_id=9, pad_type_id=0)
    exp = oracle_rows(ids, rp, js, tr, pd, True)
    monkeypatch.setenv("B2T_CHUNK_BYTES", "65536")   # many chunks through the host pipeline
    tok = Tokenizer.from_str(js)
    same(engine_rows(tok, pairs, tr, pd), exp, "fixed length, 64 KiB chunks")
    exp2 = oracle_rows(ids, rp, js, tr2, pd2, True)
    assert not isinstance(exp2, str)
    same(engine_rows(tok, pairs, tr2, pd2), exp2, "BatchLongest (one device pass)")
    # b2t_encode_pairs_dense_device
    data, off = helpers.pack_docs([s for p in pairs for s in p])
    L = _lib.lib()
    cudart = ctypes.CDLL("libcudart.so")
    for trd, pdd, e in ((tr, pd, exp), (tr2, pd2, exp2)):
        _apply(tok, trd, pdd)
        sp, keep = tok.pair_dense_spec()
        d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        res = ctypes.c_void_p()
        _lib.check(L.b2t_encode_pairs_dense_device(tok.handle, d_bytes.data_ptr(), len(data), d_off.data_ptr(), len(pairs), ctypes.byref(sp), None, ctypes.byref(res)))
        torch.cuda.synchronize()
        W, n = L.b2t_result_dense_length(res), len(pairs)
        assert L.b2t_result_on_device(res) == 1 and L.b2t_result_n_docs(res) == n and W == e[0].shape[1]

        def dev(ptr, count, dtype):
            out = np.empty(count, dtype=dtype)
            assert cudart.cudaMemcpy(ctypes.c_void_p(out.ctypes.data), ctypes.c_void_p(ptr), ctypes.c_size_t(out.nbytes), 2) == 0
            return out
        got = (dev(L.b2t_result_dense_ids(res), n * W, np.uint32).reshape(n, W), dev(L.b2t_result_type_ids(res), n * W, np.uint8).reshape(n, W),
               dev(L.b2t_result_attention_mask(res), n * W, np.uint8).reshape(n, W), dev(L.b2t_result_row_lengths(res), n, np.uint32))
        L.b2t_result_free(res)
        same(got, e, "device entry point")
    # a single-sequence result has no type ids
    _apply(tok, tr, dict(length=64, direction="right", pad_id=0, pad_type_id=0))
    res = ctypes.c_void_p()
    sp, keep = tok.dense_spec()
    _lib.check(L.b2t_encode_batch_dense(tok.handle, data.ctypes.data, off.ctypes.data, 4, ctypes.byref(sp), ctypes.byref(res)))
    assert not L.b2t_result_type_ids(res)
    L.b2t_result_free(res)


@pytest.mark.gpu
def test_gpu_pairs_device_added_tokens_and_bert_pipeline():
    from tokenizers_b200 import Tokenizer
    # added tokens extracted on the device inside both sequences of a pair
    js = json.loads(helpers.with_added_tokens(helpers.asset_json("gpt2_style")))
    js["post_processor"] = TEMPLATES["roberta"][1](js["model"]["vocab"])
    js = json.dumps(js)
    tok, ref = Tokenizer.from_str(js), helpers.oracle_backed_tokenizer(js)
    assert tok._dev_added
    docs = helpers.added_token_docs(5, 400)
    pairs = list(zip(docs[0::2], docs[1::2]))
    data, off = helpers.pack_docs([s for p in pairs for s in p])
    be, _ = ref._encode_core(data, off, 0, True)
    tr, pd = dict(max_length=48, strategy="longest_first", direction="left"), dict(length=None, direction="right", pad_id=0, pad_type_id=1)
    got = engine_rows(tok, pairs, tr, pd)
    same(got, oracle_rows(be.ids, be.row_ptr, js, tr, pd, True), "device added tokens")
    if tk is not None:
        same(got, wheel_rows(js, pairs, tr, pd, True), "device added tokens, wheel")
    # the bert-base pipeline: BertNormalizer + BertPreTokenizer + WordPiece + BertProcessing
    j = json.loads(helpers.bert_json(helpers.BERT_UNCASED))
    j["post_processor"] = TEMPLATES["bert"][1](j["model"]["vocab"])
    js = json.dumps(j)
    tok = Tokenizer.from_str(js)
    for tr, pd in SETTINGS[:3]:
        pairs = arrange([(a.upper() + " Àé 中文", b) for a, b in pairs_for(21)], tr)
        ids, rp = oracle_csr(js, pairs)
        got = engine_rows(tok, pairs, tr, pd)
        same(got, oracle_rows(ids, rp, js, tr, pd, True), ("bert", tr))
        if tk is not None:
            same(got, wheel_rows(js, pairs, tr, pd, True), ("bert", tr, "wheel"))


@pytest.mark.gpu
def test_gpu_pairs_errors_empty_batch_and_encode_batch():
    from tokenizers_b200 import Tokenizer, UnsupportedConfig, B2TError, _lib
    js = tokenizer_json("bert")
    tok = Tokenizer.from_str(js)
    pairs = pairs_for(13)
    a, b, tr = ERROR_CASES[0]
    _apply(tok, tr, SETTINGS[0][1])
    with pytest.raises(ValueError, match="too short to respect"):
        tok.encode_pairs_dense(pairs + [(a, b)])
    _apply(tok, None, dict(length=8, direction="right", pad_id=0, pad_type_id=0))
    with pytest.raises(B2TError):   # a row that does not fit a fixed length is an error, not a silently cut row
        tok.encode_pairs_dense(pairs)
    _apply(tok, dict(max_length=32, strategy="longest_first", direction="right", stride=2), SETTINGS[0][1])
    with pytest.raises(UnsupportedConfig):
        tok.encode_pairs_dense(pairs)
    j = json.loads(tokenizer_json("b_first"))
    j["post_processor"]["pair"][1]["Sequence"]["type_id"] = 256
    tok2 = Tokenizer.from_str(json.dumps(j))
    _apply(tok2, None, SETTINGS[0][1])
    with pytest.raises(UnsupportedConfig):
        tok2.encode_pairs_dense(pairs)
    _apply(tok, *SETTINGS[0])
    data, off = helpers.pack_docs([s for p in pairs for s in p])
    with pytest.raises(ValueError):   # not 2n + 1 offsets
        tok.encode_pairs_dense(data, off[:-1])
    bad = off.copy(); bad[3], bad[4] = bad[4], bad[3] + 1
    with pytest.raises(B2TError) as ei:
        tok.encode_pairs_dense(data, bad)
    assert ei.value.code == _lib.B2T_ERR_INVALID
    got = tok.encode_pairs_dense([])
    assert got["input_ids"].shape == (0, 40) and got["token_type_ids"].shape == (0, 40)
    # encode_batch on the pairs (the per-input path) stacked == the dense rows
    for name in TEMPLATES:
        js = tokenizer_json(name)
        t = Tokenizer.from_str(js)
        for tr, pd in (SETTINGS[1], SETTINGS[2]):
            pairs = arrange(pairs_for(13), tr)
            _apply(t, tr, pd)
            encs = t.encode_batch(pairs)
            n = len(pairs)
            stacked = (np.array([e.ids for e in encs], dtype=np.uint32).reshape(n, -1), np.array([e.type_ids for e in encs], dtype=np.uint8).reshape(n, -1),
                       np.array([e.attention_mask for e in encs], dtype=np.uint8).reshape(n, -1), np.array([sum(e.attention_mask) for e in encs], dtype=np.uint32))
            same(engine_rows(t, pairs, tr, pd), stacked, (name, tr, "encode_batch"))
