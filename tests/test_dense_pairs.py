"""Dense mode for pairs of sequences (b2t_encode_pairs_dense*): pair truncation, the pair template with type ids, padding.
CPU: the plain restatement (dense_oracle.dense_pair_rows) against the reference wheel and the committed fixture, the pair
kernels' own truncation algebra (dense_kernels.cuh pair_keep, compiled for the host by tests/native/dense_emul.cpp) against
the restatement on every small input, the length passes and the plain row kernels of single sequences and pairs, run on the
host, against the restatements, and the spec the shim builds.  GPU: the engine against all of them."""
import ctypes, json
import numpy as np
import pytest
import helpers, corpus
import dense_cases as dc
import dense_oracle as do
from dense_cases import tk, STRATEGIES, TOO_SHORT
from oracle import oracle as orc

SETTINGS = dc.PAIR_SETTINGS
F = dc.fields(4)   # ids, type ids, mask, lengths


def pieces_of(js, add_special_tokens):
    from tokenizers_b200.tokenizer import parse_post_processor
    tp = parse_post_processor(json.loads(js).get("post_processor"))
    pieces = [("seq", 0, 0), ("seq", 1, 1)] if tp is None else tp["pair"]
    return [p for p in pieces if p[0] == "seq" or add_special_tokens]


def oracle_rows(ids, rp, js, tr, pd, add_special_tokens):
    """dense_oracle.dense_pair_rows with the settings -> (ids, type ids, mask, lengths) or the error message"""
    try:
        return do.dense_pair_rows(ids, rp, length=pd["length"] or 0, pad_to_multiple_of=pd.get("pad_to_multiple_of") or 0,
                                  max_length=tr["max_length"] if tr else 0, strategy=tr["strategy"] if tr else "longest_first",
                                  truncate_left=bool(tr and tr["direction"] == "left"), pad_id=pd["pad_id"], pad_type_id=pd["pad_type_id"],
                                  pad_left=pd["direction"] == "left", pieces=pieces_of(js, add_special_tokens))
    except ValueError as ex:
        return str(ex)


def oracle_csr(js, pairs):
    ids, _, _, rp = orc.Oracle(js).encode_batch([s for p in pairs for s in p])
    return ids, rp


# ------------------------------------------------------------------------------------------------------------- CPU
def test_settings_reach_their_cases():
    """the settings cut with every strategy, hit budget 0 and the SequenceTooShort error on the test pairs"""
    js = dc.tokenizer_json("bert")
    for tr, _ in SETTINGS:
        tr = dc.resolve(js, tr)
        if tr is None:
            continue
        ids, rp = oracle_csr(js, dc.arrange(dc.pairs_for(11), tr))
        lens = np.diff(rp.astype(np.int64)).reshape(-1, 2)
        budget = tr["max_length"] - dc.n_special(js)
        kept = [do.pair_keep(int(a), int(b), budget, tr["strategy"]) for a, b in lens]
        assert all(k is not None for k in kept) and any(k != (a, b) for k, (a, b) in zip(kept, lens.tolist())), tr
    assert do.pair_keep(6, 2, 1, "only_first") is None and do.pair_keep(6, 0, 0, "only_first") == (0, 0)


def test_pair_keep_kernel_algebra_exhaustive():
    """dense_kernels.cuh pair_keep == the restatement for every n1, n2, budget in [0, 48] and every strategy (which inputs
    fail included), and with no truncation at all"""
    L = dc.emul()
    r = np.arange(49, dtype=np.uint32)
    n1, n2, bud = (a.reshape(-1) for a in np.meshgrid(r, r, np.append(r, np.uint32(0xFFFFFFFF)), indexing="ij"))
    for s, name in enumerate(STRATEGIES):
        st = np.full(n1.size, s, dtype=np.uint32)
        k1, k2, ok = np.zeros_like(n1), np.zeros_like(n1), np.zeros(n1.size, dtype=np.uint8)
        L.b2t_emul_pair_keep(n1.size, n1.ctypes.data, n2.ctypes.data, bud.ctypes.data, st.ctypes.data, k1.ctypes.data, k2.ctypes.data, ok.ctypes.data)
        for i in range(n1.size):
            b = int(bud[i])
            exp = do.pair_keep(int(n1[i]), int(n2[i]), None if b == 0xFFFFFFFF else b, name)
            got = (int(k1[i]), int(k2[i])) if ok[i] else None
            assert got == exp, (name, int(n1[i]), int(n2[i]), b, got, exp)
        assert not ok.all() or s == 0   # the only_* strategies do fail on some inputs


TIGHT = 8   # a fixed row length some rows of the grid do not fit


def pair_rows_at(ids, rp, width, **kw):
    """dense_pair_rows at the fixed length `width`, one pair at a time; a pair whose row does not fit is all zeros (the
    pair kernel leaves it unwritten)"""
    rows = []
    for p in range((len(rp) - 1) // 2):
        try:
            rows.append(do.dense_pair_rows(ids, rp[2 * p:2 * p + 3], length=width, pad_to_multiple_of=0, **kw))
        except ValueError as ex:
            assert "dense length" in str(ex), ex
            rows.append((np.zeros((1, width), np.uint32), np.zeros((1, width), np.uint8), np.zeros((1, width), np.uint8), np.zeros(1, np.uint32)))
    return tuple(np.concatenate(f) for f in zip(*rows))


def on_the_left(rows):
    """rows padded on the right -> the same rows padded on the left (every field's padding is one value per field)"""
    if isinstance(rows, str):
        return rows
    w = rows[0].shape[1]
    return tuple(np.stack([np.roll(x[r], w - int(n), axis=0) for r, n in enumerate(rows[3])]) if x.ndim > 1 else x for x in rows)


def test_plain_row_and_length_kernels_match_restatements():
    """the length passes without overflowing parts (row_len_max_kernel, pair_len_max_kernel) and the <0, 0, 0> / <0, 1, 0>
    row kernels of single sequences and pairs, run on the host, == oracle.dense_rows, dense_pair_rows and the kept rows of
    dense_meta_rows (offset rows) on batches of every (n1, n2) of NS, for every budget in [0, 48], every strategy, both
    directions and both padding sides (SequenceTooShort included); single sequences of every length in [0, 40] likewise.
    At a fixed length too short for some rows the single-sequence kernel raises bit 0 and cuts the row, and the pair
    kernel leaves the row unwritten."""
    L = dc.emul()
    pb, sb = dc.plain_batch([n for a in dc.NS for b in dc.NS for n in (a, b)]), dc.plain_batch(list(range(41)))
    single = dc.single_template(dc.EMUL_TEMPLATES["a_first"], 3)   # pre A post
    pre, post = [single[0][1]], [single[2][1]]
    for budget in range(49):
        for left in (False, True):
            offs = dc.restated_rows(sb, False, single, budget, "longest_first", 0, left, over=False)
            for pad_left in (False, True):
                what = (budget, left, pad_left)
                args = dict(pad_id=7, truncate_left=left, pad_left=pad_left, pre=pre, post=post)
                exp = orc.dense_rows(sb[0][:-1], sb[3], length=0, pad_to_multiple_of=0, max_length=budget + 2, **args)
                got = dc.emul_rows(L, sb, False, single, budget, 0, 0, left, over=False, offs=False, pad_left=pad_left)
                dc.same(got, (exp[0], None, exp[1], exp[2]), what + ("single",), F)
                got = dc.emul_rows(L, sb, False, single, budget, 0, 0, left, over=False, pad_left=pad_left)
                dc.same(got, on_the_left(offs) if pad_left else offs, what + ("single", "offsets"), dc.fields(6))
                exp = orc.dense_rows(sb[0][:-1], sb[3], length=TIGHT, pad_to_multiple_of=0, max_length=2 + min(budget, TIGHT - 2), **args)
                cut = int(any(min(n, budget) + 2 > TIGHT for n in range(41)))
                got = dc.emul_rows(L, sb, False, single, budget, 0, 0, left, over=False, offs=False, pad_left=pad_left, width=TIGHT, err=cut)
                dc.same(got, (exp[0], None, exp[1], exp[2]), what + ("single", "cut"), F)
            for order, pieces in dc.EMUL_TEMPLATES.items():
                n_sp = sum(1 for p in pieces if p[0] == "special")
                for strategy in range(3):
                    offs = dc.restated_rows(pb, True, pieces, budget, STRATEGIES[strategy], 0, left, over=False)
                    for pad_left in (False, True):
                        what = (order, budget, STRATEGIES[strategy], left, pad_left)
                        args = dict(max_length=budget + n_sp, strategy=STRATEGIES[strategy], truncate_left=left, pad_id=7, pad_type_id=5,
                                    pad_left=pad_left, pieces=pieces)
                        try:
                            exp = do.dense_pair_rows(pb[0][:-1], pb[3], length=0, pad_to_multiple_of=0, **args)
                        except ValueError as ex:
                            exp = str(ex)
                        got = dc.emul_rows(L, pb, True, pieces, budget, strategy, 0, left, over=False, offs=False, pad_left=pad_left)
                        dc.same(got, exp, what, F)
                        got = dc.emul_rows(L, pb, True, pieces, budget, strategy, 0, left, over=False, pad_left=pad_left)
                        dc.same(got, on_the_left(offs) if pad_left else offs, what + ("offsets",), dc.fields(6))
                        if not isinstance(exp, str):
                            got = dc.emul_rows(L, pb, True, pieces, budget, strategy, 0, left, over=False, offs=False, pad_left=pad_left, width=TIGHT)
                            dc.same(got, pair_rows_at(pb[0][:-1], pb[3], TIGHT, **args), what + ("cut",), F)


@pytest.mark.skipif(tk is None, reason="reference wheel not importable")
@pytest.mark.parametrize("name", dc.PAIR_NAMES)
def test_dense_pair_rows_matches_wheel(name):
    js = dc.tokenizer_json(name)
    for key, tr, pd, ast in dc.pair_cases():
        tr = dc.resolve(js, tr)
        pairs = dc.arrange(dc.pairs_for(11), tr)
        dc.same(oracle_rows(*oracle_csr(js, pairs), js, tr, pd, ast), dc.wheel_rows(js, pairs, tr, pd, ast), (name, key), F)


@pytest.mark.parametrize("name", dc.PAIR_NAMES)
def test_dense_pair_rows_matches_golden(name):
    """the same restatement against committed vectors of the wheel (no wheel needed)"""
    g = dc.golden("dense_pairs")
    js = dc.tokenizer_json(name)
    for key, tr, pd, ast in dc.pair_cases():
        c = g["cases"].get(f"{name}/{key}")
        tr = dc.resolve(js, tr)
        if c is None:
            assert tr is None
            continue
        pairs = dc.arrange([tuple(p) for p in g["pairs"]], tr)
        dc.same(oracle_rows(*oracle_csr(js, pairs), js, tr, pd, ast), dc.golden_rows(c), (name, key), F)
    for k, (a, b, tr) in enumerate(dc.ERROR_CASES):
        dc.same(oracle_rows(*oracle_csr(js, [(a, b)]), js, tr, SETTINGS[0][1], True), dc.golden_rows(g["cases"][f"{name}/error{k}"]), (name, k), F)


def spec_rows(tok, ids, rp, add_special_tokens):
    """the b2t_pair_dense_spec the shim builds, fed to the restatement"""
    sp, keep = tok.pair_dense_spec(add_special_tokens)
    from tokenizers_b200 import _lib
    pids, ptypes = keep
    pieces = [("seq", 0 if i == _lib.PIECE_A else 1, int(t)) if i in (_lib.PIECE_A, _lib.PIECE_B) else ("special", int(i), int(t))
              for i, t in zip(pids.tolist(), ptypes.tolist())]
    assert sp.n_pieces == len(pieces) and sp.struct_size == ctypes.sizeof(_lib.PairDenseSpec)
    try:
        return do.dense_pair_rows(ids, rp, length=sp.length, pad_to_multiple_of=sp.pad_to_multiple_of, max_length=sp.max_length,
                                  strategy=STRATEGIES[sp.strategy], truncate_left=bool(sp.truncate_left), pad_id=sp.pad_id,
                                  pad_type_id=sp.pad_type_id, pad_left=bool(sp.pad_left), pieces=pieces)
    except ValueError as ex:
        return str(ex)


@pytest.mark.parametrize("name", dc.PAIR_NAMES)
def test_pair_dense_spec_matches_wheel(name):
    """Tokenizer.pair_dense_spec (the shim's settings -> b2t_pair_dense_spec), read back into the restatement, gives the
    reference's rows: the committed vectors always, the wheel when it is importable"""
    js = dc.tokenizer_json(name)
    tok = helpers.oracle_backed_tokenizer(js)
    g = dc.golden("dense_pairs")
    for key, tr, pd, ast in dc.pair_cases():
        tr = dc.resolve(js, tr)
        if tr is None and SETTINGS[int(key.split("/")[0])][0] is not None:
            continue
        dc.apply(tok, tr, pd)
        gpairs = dc.arrange([tuple(p) for p in g["pairs"]], tr)
        dc.same(spec_rows(tok, *oracle_csr(js, gpairs), ast), dc.golden_rows(g["cases"][f"{name}/{key}"]), (name, key, "golden"), F)
        if tk is not None:
            pairs = dc.arrange(dc.pairs_for(11), tr)
            dc.same(spec_rows(tok, *oracle_csr(js, pairs), ast), dc.wheel_rows(js, pairs, tr, pd, ast), (name, key, "wheel"), F)


def test_pair_dense_spec_refusals():
    from tokenizers_b200 import UnsupportedConfig
    js = json.loads(dc.tokenizer_json("b_first"))
    tok = helpers.oracle_backed_tokenizer(json.dumps(js))
    dc.apply(tok, dict(max_length=32, strategy="longest_first", direction="right", stride=4), SETTINGS[0][1])
    with pytest.raises(UnsupportedConfig):   # overflowing parts have no dense form
        tok.pair_dense_spec()
    dc.apply(tok, dict(max_length=3, strategy="longest_first", direction="right"), SETTINGS[0][1])
    with pytest.raises(ValueError):          # max_length below the 5 special tokens of the pair template
        tok.pair_dense_spec()
    tok.no_padding()
    with pytest.raises(UnsupportedConfig):
        tok.pair_dense_spec()
    js["post_processor"]["pair"] = []          # a template without a pair form
    tok = helpers.oracle_backed_tokenizer(json.dumps(js))
    dc.apply(tok, None, SETTINGS[0][1])
    with pytest.raises(ValueError, match="no template for pairs"):
        tok.pair_dense_spec()


# ------------------------------------------------------------------------------------------------------------- GPU
def engine_rows(tok, pairs, tr, pd, add_special_tokens=True):
    dc.apply(tok, tr, pd)
    try:
        out = tok.encode_pairs_dense(pairs, add_special_tokens=add_special_tokens)
    except ValueError as ex:
        if TOO_SHORT not in str(ex):
            raise
        return str(ex)
    return out["input_ids"], out["token_type_ids"], out["attention_mask"], out["lengths"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", dc.PAIR_NAMES)
def test_gpu_pairs_match_oracle_wheel_and_golden(name):
    from tokenizers_b200 import Tokenizer
    js = dc.tokenizer_json(name)
    tok = Tokenizer.from_str(js)
    g = dc.golden("dense_pairs")
    for key, tr, pd, ast in dc.pair_cases():
        tr0, tr = tr, dc.resolve(js, tr)
        if tr is None and tr0 is not None:
            continue
        pairs, gpairs = dc.arrange(dc.pairs_for(12), tr), dc.arrange([tuple(p) for p in g["pairs"]], tr)
        got = engine_rows(tok, pairs, tr, pd, ast)
        dc.same(got, oracle_rows(*oracle_csr(js, pairs), js, tr, pd, ast), (name, key, "oracle"), F)
        if tk is not None:
            dc.same(got, dc.wheel_rows(js, pairs, tr, pd, ast), (name, key, "wheel"), F)
        dc.same(engine_rows(tok, gpairs, tr, pd, ast), dc.golden_rows(g["cases"][f"{name}/{key}"]), (name, key, "golden"), F)
    for k, (a, b, tr) in enumerate(dc.ERROR_CASES):   # SequenceTooShort: the whole batch fails with the reference's message
        dc.apply(tok, tr, SETTINGS[0][1])
        with pytest.raises(ValueError, match="too short"):
            tok.encode_pairs_dense(dc.pairs_for(12)[:5] + [(a, b)])


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
    js = dc.tokenizer_json("roberta")
    pairs = chunk_pairs()
    ids, rp = oracle_csr(js, pairs)
    tr, pd = dict(max_length=64, strategy="longest_first", direction="right"), dict(length=64, direction="right", pad_id=9, pad_type_id=1)
    tr2, pd2 = dict(max_length=100, strategy="longest_first", direction="left"), dict(length=None, direction="left", pad_id=9, pad_type_id=0)
    exp = oracle_rows(ids, rp, js, tr, pd, True)
    monkeypatch.setenv("B2T_CHUNK_BYTES", "65536")   # many chunks through the host pipeline
    tok = Tokenizer.from_str(js)
    dc.same(engine_rows(tok, pairs, tr, pd), exp, "fixed length, 64 KiB chunks", F)
    exp2 = oracle_rows(ids, rp, js, tr2, pd2, True)
    assert not isinstance(exp2, str)
    dc.same(engine_rows(tok, pairs, tr2, pd2), exp2, "BatchLongest (one device pass)", F)
    # b2t_encode_pairs_dense_device
    data, off = helpers.pack_docs([s for p in pairs for s in p])
    L = _lib.lib()
    cudart = ctypes.CDLL("libcudart.so")
    for trd, pdd, e in ((tr, pd, exp), (tr2, pd2, exp2)):
        dc.apply(tok, trd, pdd)
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
        dc.same(got, e, "device entry point", F)
    # a single-sequence result has no type ids
    dc.apply(tok, tr, dict(length=64, direction="right", pad_id=0, pad_type_id=0))
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
    js["post_processor"] = dc.TEMPLATES["roberta"][1](js["model"]["vocab"])
    js = json.dumps(js)
    tok, ref = Tokenizer.from_str(js), helpers.oracle_backed_tokenizer(js)
    assert tok._dev_added
    docs = helpers.added_token_docs(5, 400)
    pairs = list(zip(docs[0::2], docs[1::2]))
    data, off = helpers.pack_docs([s for p in pairs for s in p])
    be, _ = ref._encode_core(data, off, 0, True)
    tr, pd = dict(max_length=48, strategy="longest_first", direction="left"), dict(length=None, direction="right", pad_id=0, pad_type_id=1)
    got = engine_rows(tok, pairs, tr, pd)
    dc.same(got, oracle_rows(be.ids, be.row_ptr, js, tr, pd, True), "device added tokens", F)
    if tk is not None:
        dc.same(got, dc.wheel_rows(js, pairs, tr, pd, True), "device added tokens, wheel", F)
    # the bert-base pipeline: BertNormalizer + BertPreTokenizer + WordPiece + BertProcessing
    j = json.loads(helpers.bert_json(helpers.BERT_UNCASED))
    j["post_processor"] = dc.TEMPLATES["bert"][1](j["model"]["vocab"])
    js = json.dumps(j)
    tok = Tokenizer.from_str(js)
    for tr, pd in SETTINGS[:3]:
        pairs = dc.arrange([(a.upper() + " Àé 中文", b) for a, b in dc.pairs_for(21)], tr)
        ids, rp = oracle_csr(js, pairs)
        got = engine_rows(tok, pairs, tr, pd)
        dc.same(got, oracle_rows(ids, rp, js, tr, pd, True), ("bert", tr), F)
        if tk is not None:
            dc.same(got, dc.wheel_rows(js, pairs, tr, pd, True), ("bert", tr, "wheel"), F)


@pytest.mark.gpu
def test_gpu_pairs_errors_empty_batch_and_encode_batch():
    from tokenizers_b200 import Tokenizer, UnsupportedConfig, B2TError, _lib
    js = dc.tokenizer_json("bert")
    tok = Tokenizer.from_str(js)
    pairs = dc.pairs_for(13)
    a, b, tr = dc.ERROR_CASES[0]
    dc.apply(tok, tr, SETTINGS[0][1])
    with pytest.raises(ValueError, match="too short to respect"):
        tok.encode_pairs_dense(pairs + [(a, b)])
    dc.apply(tok, None, dict(length=8, direction="right", pad_id=0, pad_type_id=0))
    with pytest.raises(B2TError):   # a row that does not fit a fixed length is an error, not a silently cut row
        tok.encode_pairs_dense(pairs)
    dc.apply(tok, dict(max_length=32, strategy="longest_first", direction="right", stride=2), SETTINGS[0][1])
    with pytest.raises(UnsupportedConfig):
        tok.encode_pairs_dense(pairs)
    j = json.loads(dc.tokenizer_json("b_first"))
    j["post_processor"]["pair"][1]["Sequence"]["type_id"] = 256
    tok2 = Tokenizer.from_str(json.dumps(j))
    dc.apply(tok2, None, SETTINGS[0][1])
    with pytest.raises(UnsupportedConfig):
        tok2.encode_pairs_dense(pairs)
    dc.apply(tok, *SETTINGS[0])
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
    for name in dc.PAIR_NAMES:
        js = dc.tokenizer_json(name)
        t = Tokenizer.from_str(js)
        for tr, pd in (SETTINGS[1], SETTINGS[2]):
            pairs = dc.arrange(dc.pairs_for(13), tr)
            dc.apply(t, tr, pd)
            encs = t.encode_batch(pairs)
            n = len(pairs)
            stacked = (np.array([e.ids for e in encs], dtype=np.uint32).reshape(n, -1), np.array([e.type_ids for e in encs], dtype=np.uint8).reshape(n, -1),
                       np.array([e.attention_mask for e in encs], dtype=np.uint8).reshape(n, -1), np.array([sum(e.attention_mask) for e in encs], dtype=np.uint32))
            dc.same(engine_rows(t, pairs, tr, pd), stacked, (name, tr, "encode_batch"), F)
