"""Dense rows with the per-position metadata of the reference's post-processed Encoding (B2T_DENSE_TRIM_OFFSETS,
B2T_DENSE_SPECIAL_MASK, B2T_DENSE_SEQUENCE_IDS, B2T_DENSE_WORD_IDS): offsets trimmed by ByteLevel process_offsets on every
part of every sequence, the special-tokens mask, sequence ids and word ids.
CPU: the trim rules of dense_kernels.cuh (trim_span, added_trim_counts) and its META row kernels, run on the host by
tests/native/dense_emul.cpp, against the shim's host restatement (trim_spans, _span_spaces, pairs.post_process); that
restatement (dense_oracle.dense_meta_rows) against the reference wheel and the committed fixture; the spec the shim builds.
GPU: the engine against all of them."""
import ctypes, json, random
import numpy as np
import pytest
import helpers
import dense_cases as dc
import dense_oracle as do
from dense_cases import tk, PANIC, TOO_SHORT, NOT_FIT, flat
from tokenizers_b200.tokenizer import parse_post_processor, trim_spans

SETTINGS = dc.META_SETTINGS


def fields(is_pair=True, seq=True):
    """the nine fields; type ids where the engine returns them; seq = False: not the sequence ids (the tokenizer without a
    post-processor, whose sequence ids dense mode refuses)"""
    return dc.fields(9, is_pair, seq=seq)


def oracle_rows(js, inputs, tr, pd, over, is_pair, ast):
    """dense_oracle.dense_meta_rows on the CSR (ids, offsets, words) and space counts the shim's host logic gives in front of
    the oracle"""
    from tokenizers_b200 import _lib
    ref = helpers.oracle_backed_tokenizer(js)
    data, off = helpers.pack_docs(flat(inputs))
    be, trim = ref._encode_core(data, off, _lib.WANT_OFFSETS | _lib.WANT_WORD_IDS, True)
    tp = parse_post_processor(json.loads(js).get("post_processor"))
    ld, trl = trim if trim is not None else (None, None)
    out = do.dense_meta_rows(be.ids, be.offsets, be.word_ids, be.row_ptr, ld, trl, is_pair=is_pair, template=tp, truncation=tr, padding=pd,
                             add_special_tokens=ast)
    return out if isinstance(out, str) or over else dc.kept_rows(out)


# ------------------------------------------------------------------------------------------------------------- CPU
def test_trim_span_exhaustive():
    """trim_span == trim_spans (ByteLevel process_offsets) for every o0 <= o1 <= 12, ld, tr <= 6, first and add_prefix_space"""
    L = dc.emul()
    out = (ctypes.c_uint32 * 2)()
    cases = [(o0, o1, ld, tr, f, a) for o1 in range(13) for o0 in range(o1 + 1) for ld in range(7) for tr in range(7) for f in (0, 1) for a in (0, 1)]
    c = np.asarray(cases, dtype=np.int64)
    for aps in (False, True):
        sel = c[c[:, 5] == int(aps)]
        exp = trim_spans(sel[:, :2], sel[:, 2], sel[:, 3], sel[:, 4].astype(bool), aps)
        for row, e in zip(sel.tolist(), exp.tolist()):
            L.b2t_emul_trim_span(*row[:4], row[4], row[5], out)
            assert [out[0], out[1]] == e, row


def _rust_space_table():
    from tokenizers_b200 import _lib
    tbl = np.zeros(0x110000, dtype=np.uint8)
    _lib.check(_lib.lib().b2t_unicode_class_table(1, tbl.ctypes.data))
    return tbl


def _span_spaces(text, cls):
    """Tokenizer._span_spaces on a text: leading / trailing chars that are whitespace (Rust \\s) or U+0120"""
    from tokenizers_b200 import added
    ws = lambda ch: ch == "Ġ" or cls[ord(ch)] == added.CLS_S
    lead = next((k for k, ch in enumerate(text) if not ws(ch)), len(text))
    trail = next((k for k, ch in enumerate(reversed(text)) if not ws(ch)), len(text))
    return lead, trail


def _entry(content, cls):
    """the engine's per-added-token entry of a content: (chars, lead, trail, TRIM_ALL_SPACE)"""
    lead, trail = _span_spaces(content, cls)
    return len(content), lead, trail, 1 if lead == len(content) else 0


SPACES = [" ", "\t", "\n", "\u0085", " ", " ", "　"]
CONTENTS = ["<mask>", " <x>", "<y>　", "ĠtokĠ", "ĠĠ", " ", "  ", "a b", "Ġ x \n", "z\u0085"]


def test_added_trim_counts_match_span_spaces():
    """added_trim_counts == _span_spaces on the span a match makes (absorbed whitespace left for lstrip, right for rstrip)
    for every flag set, contents that start or end with whitespace or U+0120, all-whitespace contents, ASCII and
    non-ASCII White_Space; ambiguous exactly when both flags are set and the span is longer than the content"""
    L = dc.emul()
    cls = _rust_space_table()
    rng = random.Random(5)
    ld, tr = ctypes.c_uint32(), ctypes.c_uint32()
    n_amb = 0
    for content in CONTENTS:
        chars, lc, tc, allws = _entry(content, cls)
        for lstrip in (False, True):
            for rstrip in (False, True):
                flags = allws | (2 if lstrip else 0) | (4 if rstrip else 0)
                for _ in range(12):
                    left = "".join(rng.choice(SPACES) for _ in range(rng.randint(0, 3))) if lstrip else ""
                    right = "".join(rng.choice(SPACES) for _ in range(rng.randint(0, 3))) if rstrip else ""
                    span = left + content + right
                    ok = L.b2t_emul_added_trim_counts(len(span), chars, lc, tc, flags, ctypes.byref(ld), ctypes.byref(tr))
                    amb = lstrip and rstrip and len(span) > chars
                    assert ok == (0 if amb else 1), (content, lstrip, rstrip, span)
                    n_amb += amb
                    if ok:
                        assert (ld.value, tr.value) == _span_spaces(span, cls), (content, lstrip, rstrip, span)
    assert n_amb > 0


def emul_batch(lens, seed):
    """a CSR of documents with `lens` tokens: token t of document d has id 1000 d + t (every 7th one an added token: bit 31,
    one of ADDED), words t // 2, offsets that leave gaps; -> (ids, offsets, words, row_ptr, trim_vocab, added entries, ld, tr)
    where ld / tr are the restatement's counts: the vocabulary's, and _span_spaces on the span text of an added token"""
    rng = random.Random(seed)
    cls = _rust_space_table()
    added = [(500 + k, c, ls, rs) for k, (c, ls, rs) in enumerate([("<m>", True, False), ("[s]", False, True), ("<b>", True, True),
                                                                        (" <w>", True, False), ("ĠĠ", False, True)])]
    n_ids = 1000 * len(lens) + 1
    vocab_ld = np.array([rng.choice([0, 0, 1, 2, 3]) for _ in range(n_ids)], dtype=np.uint32)
    vocab_tr = np.array([rng.choice([0, 0, 0, 1, 2]) for _ in range(n_ids)], dtype=np.uint32)
    ids, offs, words, ld, tr = [], [], [], [], []
    for d, n in enumerate(lens):
        pos = rng.randint(0, 1)
        for t in range(n):
            w = rng.randint(1, 5)
            if t % 7 == 3:
                aid, content, ls, rs = rng.choice(added)
                left = "".join(rng.choice(SPACES) for _ in range(rng.randint(0, 2))) if ls and not rs else ""
                right = "".join(rng.choice(SPACES) for _ in range(rng.randint(0, 2))) if rs and not ls else ""
                span = left + content + right
                ids.append(aid | 0x80000000); a, b = _span_spaces(span, cls); w = len(span)
            else:
                ids.append(1000 * d + t); a, b = int(vocab_ld[1000 * d + t]), int(vocab_tr[1000 * d + t])
            offs.append((pos, pos + w)); words.append(t // 2); ld.append(a); tr.append(b)
            pos += w + rng.randint(0, 1)
    rp = np.zeros(len(lens) + 1, dtype=np.uint64); np.cumsum(lens, out=rp[1:])
    entries = sorted((aid, *_entry(c, cls)[:3], _entry(c, cls)[3] | (2 if ls else 0) | (4 if rs else 0)) for aid, c, ls, rs in added)
    tab = np.asarray([[e[0], e[1], e[2] | e[3] << 16, e[4]] for e in entries], dtype=np.uint32)
    return (np.asarray(ids + [0], dtype=np.uint32), np.asarray(offs + [(0, 0)], dtype=np.uint32).reshape(-1, 2),
            np.asarray(words + [0], dtype=np.uint32), rp, (vocab_ld | vocab_tr << 16).astype(np.uint32), tab, ld, tr)


NS = (0, 1, 2, 5, 13, 30)


@pytest.mark.parametrize("order", list(dc.EMUL_TEMPLATES))
def test_meta_kernels_match_post_process(order):
    """the META row kernels (with and without overflowing parts, with both add_prefix_space rules), run on the host, ==
    dense_meta_rows' pairs.post_process: trimmed offsets with the first token of every part of X and of Y, vocabulary counts
    for plain tokens and span counts for marked added tokens, ids without the mark, special-tokens mask, sequence ids (B
    first included), word ids; single sequences likewise"""
    L = dc.emul()
    pieces = dc.EMUL_TEMPLATES[order]
    lens = [n for a in NS for b in NS for n in (a, b)]
    batch = emul_batch(lens, 3)
    sbatch = emul_batch(list(range(31)), 4)
    for budget in (0, 3, 9, 20, 48):
        for stride in sorted({0, 1, max(budget // 2 - 1, 0)}):
            for strategy in range(3):
                for left in (False, True):
                    for over in (True, False):
                        st = stride if over else 0   # (without overflowing parts the engine runs with no stride)
                        for aps in (False, True):
                            what = (order, budget, st, strategy, left, over, aps)
                            exp = dc.restated_rows(batch, True, pieces, budget, dc.STRATEGIES[strategy], st, left, over=over, trim=aps)
                            got = dc.emul_rows(L, batch, True, pieces, budget, strategy, st, left, over=over, meta=True, aps=aps)
                            dc.same(got, exp, what, fields())
                            if strategy == 0 and order == "a_first":
                                single = dc.single_template(pieces, 2)
                                exp = dc.restated_rows(sbatch, False, single, budget, "longest_first", st, left, over=over, trim=aps)
                                got = dc.emul_rows(L, sbatch, False, single, budget, 0, st, left, over=over, meta=True, aps=aps)
                                dc.same(got, exp, what + ("single",), fields(False))


def test_meta_kernels_flag_ambiguous_and_unknown_added_tokens():
    """an lstrip + rstrip added token whose span is longer than its content raises ERR_TRIM_AMBIGUOUS (128); one with
    nothing absorbed does not"""
    L = dc.emul()
    cls = _rust_space_table()
    chars, lc, tc, allws = _entry("<b>", cls)
    tab = np.asarray([[7, chars, lc | tc << 16, allws | 6]], dtype=np.uint32)
    for width, exp in ((3, 0), (4, 128)):
        ids = np.asarray([1, 7 | 0x80000000, 2, 0], dtype=np.uint32)
        offs = np.asarray([(0, 1), (1, 1 + width), (1 + width, 3 + width), (0, 0)], dtype=np.uint32)
        rp = np.asarray([0, 3], dtype=np.uint64)
        tv = np.zeros(8, np.uint32)
        out = np.zeros((1, 8), np.uint32); ooff = np.zeros((1, 8, 2), np.uint32); olen = np.zeros(2, np.uint32); m = np.zeros((1, 8), np.uint8)
        e = L.b2t_emul_dense_rows(ids.ctypes.data, offs.ctypes.data, None, rp.ctypes.data, 1, 0, 0, 1, 1, None, 1, 8, 0xFFFFFFFF, 0, 0, 0, 0, 0, 0,
                                  0, 0, 0, None, 0, 0, 0, 0, 0, tv.ctypes.data, tab.ctypes.data, 1, 0, out.ctypes.data, None, m.ctypes.data,
                                  olen.ctypes.data, None, ooff.ctypes.data, None, None, None)
        assert e == exp, (width, e)
        assert out[0, :3].tolist() == [1, 7, 2]


def test_meta_oracle_matches_wheel_and_golden():
    """the restatement == the committed vectors of the wheel on every template and setting, and == the wheel itself where
    it is importable"""
    g = dc.golden("dense_meta")
    for name in dc.META_NAMES:
        js = dc.tokenizer_json(name)
        for key, tr, pd, over, is_pair, ast in dc.meta_cases():
            inputs = dc.arrange([tuple(p) for p in g["inputs"][name]], tr, is_pair)
            o = oracle_rows(js, inputs, tr, pd, over, is_pair, ast)
            dc.same(o, dc.golden_rows(g["cases"][f"{name}/{key}"]), (name, key, "golden"), fields(is_pair, name != "none"), ref=o)
            if tk is not None:
                inputs = dc.arrange(dc.meta_inputs(name, 17), tr, is_pair)
                o = oracle_rows(js, inputs, tr, pd, over, is_pair, ast)
                dc.same(o, dc.wheel_rows(js, inputs, tr, pd, ast, over), (name, key, "wheel"), fields(is_pair, name != "none"), ref=o)


def test_golden_covers_the_trim_cases():
    """the fixture holds multi-space tokens that are trimmed, a part whose first token keeps its space only because it is
    first, added tokens trimmed by their absorbed whitespace, and both sequence ids"""
    g = dc.golden("dense_meta")
    c = g["cases"]["roberta_aps/0/pair/1"]
    seq = np.array(c["seq"])
    assert (seq == 0).any() and (seq == 1).any() and len(set(c["sample"])) < len(c["sample"])
    assert "roberta_added/3/single/0" in g["cases"] and any("<mask>" in a for a, _ in g["inputs"]["roberta_added"])


def test_meta_spec_flags_sizes_and_default_refusal():
    from tokenizers_b200 import UnsupportedConfig, _lib
    tok = helpers.oracle_backed_tokenizer(dc.tokenizer_json("roberta_aps"))
    dc.apply(tok, dict(max_length=32, strategy="only_second", direction="right", stride=4), dc.PAIR_SETTINGS[0][1])
    with pytest.raises(UnsupportedConfig):   # the default is unchanged: offsets behind trim_offsets are refused
        tok.pair_dense_spec(return_overflowing_tokens=True, return_offsets_mapping=True)
    with pytest.raises(UnsupportedConfig):
        tok.dense_spec(return_offsets_mapping=True)
    sp, _ = tok.pair_dense_spec(return_overflowing_tokens=True, return_offsets_mapping=True, trim_offsets=True)
    assert sp.dense_flags == _lib.DENSE_OVERFLOW | _lib.DENSE_OFFSETS | _lib.DENSE_TRIM_OFFSETS | _lib.DENSE_TRIM_PREFIX_SPACE
    sp, _ = tok.dense_spec(trim_offsets=True, return_special_tokens_mask=True, return_sequence_ids=True, return_word_ids=True)
    assert sp.dense_flags == _lib.DENSE_SPECIAL_MASK | _lib.DENSE_SEQUENCE_IDS | _lib.DENSE_WORD_IDS   # (no offsets: nothing to trim)
    tok = helpers.oracle_backed_tokenizer(dc.tokenizer_json("roberta"))
    dc.apply(tok, dict(max_length=32, strategy="longest_first", direction="right", stride=0), dc.PAIR_SETTINGS[0][1])
    sp, _ = tok.dense_spec(return_offsets_mapping=True, trim_offsets=True)
    assert sp.dense_flags == _lib.DENSE_OFFSETS | _lib.DENSE_TRIM_OFFSETS   # add_prefix_space false
    tok = helpers.oracle_backed_tokenizer(dc.tokenizer_json("bert"))
    dc.apply(tok, dict(max_length=32, strategy="longest_first", direction="right", stride=0), dc.PAIR_SETTINGS[0][1])
    sp, _ = tok.pair_dense_spec(return_offsets_mapping=True, trim_offsets=True, return_word_ids=True)
    assert sp.dense_flags == _lib.DENSE_OFFSETS | _lib.DENSE_WORD_IDS   # nothing trims here
    sp, _ = tok.dense_spec()
    assert (sp.dense_flags, ctypes.sizeof(sp), ctypes.sizeof(_lib.PairDenseSpec)) == (0, 72, 80)
    tok = helpers.oracle_backed_tokenizer(dc.tokenizer_json("none"))
    dc.apply(tok, dict(max_length=32, strategy="longest_first", direction="right", stride=0), dc.PAIR_SETTINGS[0][1])
    with pytest.raises(UnsupportedConfig):   # no post-processor: the reference's sequence ids follow default_process's bookkeeping
        tok.pair_dense_spec(return_sequence_ids=True)
    sp, _ = tok.pair_dense_spec(return_special_tokens_mask=True, return_word_ids=True)
    assert sp.dense_flags == _lib.DENSE_SPECIAL_MASK | _lib.DENSE_WORD_IDS
    assert (_lib.DENSE_TRIM_OFFSETS, _lib.DENSE_TRIM_PREFIX_SPACE, _lib.DENSE_SPECIAL_MASK, _lib.DENSE_SEQUENCE_IDS, _lib.DENSE_WORD_IDS) == (4, 8, 16, 32, 64)


# ------------------------------------------------------------------------------------------------------------- GPU
ALL = dict(return_special_tokens_mask=True, return_sequence_ids=True, return_word_ids=True)


def engine_rows(tok, inputs, tr, pd, over, is_pair, ast=True, **kw):
    from tokenizers_b200 import B2TError
    dc.apply(tok, tr, pd)
    kw = dict(ALL, return_sequence_ids=tok._template is not None, **kw)
    try:
        f = tok.encode_pairs_dense if is_pair else tok.encode_batch_dense
        out = f(inputs, add_special_tokens=ast, return_overflowing_tokens=over, return_offsets_mapping=True, trim_offsets=True, **kw)
    except ValueError as ex:
        if PANIC not in str(ex) and TOO_SHORT not in str(ex):
            raise
        return str(ex)
    except B2TError as ex:
        if NOT_FIT not in str(ex):
            raise
        return str(ex)
    return (out["input_ids"], out.get("token_type_ids"), out["attention_mask"], out["lengths"], out.get("overflow_to_sample_mapping"),
            out["offset_mapping"], out.get("special_tokens_mask"), out.get("sequence_ids"), out.get("word_ids"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", dc.META_NAMES)
def test_gpu_meta_matches_oracle_wheel_and_golden(name):
    from tokenizers_b200 import Tokenizer
    js = dc.tokenizer_json(name)
    tok = Tokenizer.from_str(js)
    g = dc.golden("dense_meta")
    for key, tr, pd, over, is_pair, ast in dc.meta_cases():
        inputs = dc.arrange(dc.meta_inputs(name, 18), tr, is_pair)
        got = engine_rows(tok, inputs, tr, pd, over, is_pair, ast)
        dc.same(got, oracle_rows(js, inputs, tr, pd, over, is_pair, ast), (name, key, "oracle"), fields(is_pair))
        if tk is not None:
            dc.same(got, dc.wheel_rows(js, inputs, tr, pd, ast, over), (name, key, "wheel"), fields(is_pair))
        ginputs = dc.arrange([tuple(p) for p in g["inputs"][name]], tr, is_pair)
        dc.same(engine_rows(tok, ginputs, tr, pd, over, is_pair, ast), dc.golden_rows(g["cases"][f"{name}/{key}"]), (name, key, "golden"), fields(is_pair))


def device_rows(tok, seqs, is_pair, sp):
    """the device entry points with spec sp -> the nine fields copied back from the device"""
    from tokenizers_b200 import _lib
    import torch
    L = _lib.lib()
    cudart = ctypes.CDLL("libcudart.so")

    def dev(ptr, count, dtype):
        out = np.empty(count, dtype=dtype)
        if count:
            assert cudart.cudaMemcpy(ctypes.c_void_p(out.ctypes.data), ctypes.c_void_p(ptr), ctypes.c_size_t(out.nbytes), 2) == 0
        return out
    data, off = helpers.pack_docs(flat(seqs))
    d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    res = ctypes.c_void_p()
    f = L.b2t_encode_pairs_dense_device if is_pair else L.b2t_encode_batch_dense_device
    _lib.check(f(tok.handle, d_bytes.data_ptr(), len(data), d_off.data_ptr(), len(seqs), ctypes.byref(sp), None, ctypes.byref(res)))
    torch.cuda.synchronize()
    W, R = L.b2t_result_dense_length(res), L.b2t_result_dense_rows(res)
    sample = L.b2t_result_row_sample(res)
    got = (dev(L.b2t_result_dense_ids(res), R * W, np.uint32).reshape(R, W),
           dev(L.b2t_result_type_ids(res), R * W, np.uint8).reshape(R, W) if is_pair else None,
           dev(L.b2t_result_attention_mask(res), R * W, np.uint8).reshape(R, W), dev(L.b2t_result_row_lengths(res), R, np.uint32),
           dev(sample, R, np.uint32) if sample else None, dev(L.b2t_result_dense_offsets(res), 2 * R * W, np.uint32).reshape(R, W, 2),
           dev(L.b2t_result_special_tokens_mask(res), R * W, np.uint8).reshape(R, W), dev(L.b2t_result_sequence_ids(res), R * W, np.int8).reshape(R, W),
           dev(L.b2t_result_dense_word_ids(res), R * W, np.uint32).reshape(R, W).view(np.int32))
    L.b2t_result_free(res)
    return got


@pytest.mark.gpu
def test_gpu_meta_chunks_batch_longest_and_device_entry_points(monkeypatch):
    """QA pairs (long contexts, many windows) through RoBERTa with add_prefix_space: 64 KiB chunks at a fixed length and
    BatchLongest, left / right padding and truncation, on the host path and on both device entry points"""
    from tokenizers_b200 import Tokenizer
    monkeypatch.setenv("B2T_CHUNK_BYTES", "65536")
    js = dc.tokenizer_json("roberta_aps")
    tok = Tokenizer.from_str(js)
    qa = [(q, "  " + c.replace(" ", "  ", 3)) for q, c in dc.qa_inputs()]
    for tr, pd, over in ((dict(max_length=64, stride=16, strategy="only_second", direction="right"), dict(length=64, direction="right", pad_id=1, pad_type_id=0), True),
                         (dict(max_length=48, stride=8, strategy="only_second", direction="left"), dict(length=None, direction="left", pad_id=1, pad_type_id=0), True),
                         (dict(max_length=40, stride=0, strategy="only_second", direction="right"), dict(length=40, direction="left", pad_id=1, pad_type_id=0), False)):
        for is_pair in (True, False):
            seqs = qa if is_pair else [b for _, b in qa]
            trs = tr if is_pair else dict(tr, strategy="longest_first")
            exp = oracle_rows(js, seqs, trs, pd, over, is_pair, True)
            assert not isinstance(exp, str)
            what = (trs["direction"], pd["direction"], over, is_pair)
            dc.same(engine_rows(tok, seqs, trs, pd, over, is_pair), exp, what + ("host",), fields(is_pair))
            dc.apply(tok, trs, pd)
            sp, keep = (tok.pair_dense_spec if is_pair else tok.dense_spec)(return_overflowing_tokens=over, return_offsets_mapping=True, trim_offsets=True, **ALL)
            dc.same(device_rows(tok, seqs, is_pair, sp), exp, what + ("device",), fields(is_pair))


@pytest.mark.gpu
def test_gpu_meta_added_tokens_and_both_flags_refusal():
    """device-extracted added tokens with 0, 1 and several absorbed whitespace chars, trimmed as the reference trims them;
    <both> (lstrip + rstrip) is fine while it absorbs nothing and refused (UnsupportedConfig, from both entry points and
    the device entry point) as soon as it absorbs whitespace in a row"""
    from tokenizers_b200 import Tokenizer, UnsupportedConfig, B2TError, _lib
    js = dc.tokenizer_json("roberta_added")
    tok = Tokenizer.from_str(js)
    assert tok._dev_added
    docs = ["cat<mask>", "cat <mask>", "cat   <mask>", "cat　 \t<mask> x", "[SEP2]dog", "[SEP2] dog", "[SEP2]    dog", "a<both>b", "<both>"]
    pairs = [(a, b) for a in docs for b in docs[::2]]
    for tr, pd, over in SETTINGS:
        for is_pair in (True, False):
            if not is_pair and tr is not None and tr["strategy"] == "only_second":
                continue
            seqs = dc.arrange(pairs, tr, is_pair)
            got = engine_rows(tok, seqs, tr, pd, over, is_pair)
            dc.same(got, oracle_rows(js, seqs, tr, pd, over, is_pair, True), (tr, is_pair, "oracle"), fields(is_pair))
            if tk is not None:
                dc.same(got, dc.wheel_rows(js, seqs, tr, pd, True, over), (tr, is_pair, "wheel"), fields(is_pair))
    tr, pd, _ = SETTINGS[0]
    bad = [("x <both>  y", "z"), ("a", "b")]
    with pytest.raises(UnsupportedConfig, match="lstrip and rstrip"):
        engine_rows(tok, bad, tr, pd, True, True)
    with pytest.raises(UnsupportedConfig, match="lstrip and rstrip"):
        engine_rows(tok, [a for a, _ in bad], None, dict(pd, length=None), False, False)
    with pytest.raises(B2TError, match="lstrip and rstrip") as ei:
        sp, keep = tok.pair_dense_spec(return_overflowing_tokens=True, return_offsets_mapping=True, trim_offsets=True)
        device_rows(tok, bad, True, sp)
    assert ei.value.code == _lib.B2T_ERR_UNSUPPORTED
    # without trimming the same batch goes through, and so does the engine's next call
    out = tok.encode_pairs_dense(bad, return_overflowing_tokens=True, **ALL)
    assert out["input_ids"].shape[0] == 2 and (out["sequence_ids"][0] == 1).any()


@pytest.mark.gpu
def test_gpu_trim_on_non_trimming_tokenizers_and_switches_off():
    """trim_offsets=True where the post-processor does not trim == the plain offset rows; with every new switch off the
    dicts and the raw results are byte-identical to calls without the new arguments"""
    from tokenizers_b200 import Tokenizer, _lib
    for name in ("bert", "b_first", "none"):
        tok = Tokenizer.from_str(dc.tokenizer_json(name))
        dc.apply(tok, dict(max_length=24, stride=4, strategy="longest_first", direction="right"), dict(length=32, direction="right", pad_id=0, pad_type_id=0))
        for is_pair in (True, False):
            seqs = dc.meta_inputs(name, 3) if is_pair else [a for a, _ in dc.meta_inputs(name, 3)]
            f = tok.encode_pairs_dense if is_pair else tok.encode_batch_dense
            plain = f(seqs, return_overflowing_tokens=True, return_offsets_mapping=True)
            trimmed = f(seqs, return_overflowing_tokens=True, return_offsets_mapping=True, trim_offsets=True)
            off = f(seqs, return_overflowing_tokens=True, return_offsets_mapping=True, trim_offsets=False, return_special_tokens_mask=False,
                    return_sequence_ids=False, return_word_ids=False)
            assert set(plain) == set(trimmed) == set(off)
            for k in plain:
                assert plain[k].dtype == off[k].dtype and plain[k].tobytes() == trimmed[k].tobytes() == off[k].tobytes(), (name, is_pair, k)
    # raw results: the specs with every new switch off, against the specs the shim built before these switches
    tok = Tokenizer.from_str(dc.tokenizer_json("roberta"))
    dc.apply(tok, dict(max_length=20, stride=2, strategy="longest_first", direction="left"), dict(length=None, direction="right", pad_id=0, pad_type_id=0))
    L = _lib.lib()
    for is_pair in (True, False):
        seqs = dc.meta_inputs("roberta", 4) if is_pair else [a for a, _ in dc.meta_inputs("roberta", 4)]
        data, off = helpers.pack_docs(flat(seqs))
        outs = []
        for kw in ({}, dict(trim_offsets=False, return_special_tokens_mask=False, return_sequence_ids=False, return_word_ids=False)):
            sp, keep = (tok.pair_dense_spec if is_pair else tok.dense_spec)(return_overflowing_tokens=True, **kw)
            res = ctypes.c_void_p()
            f = L.b2t_encode_pairs_dense if is_pair else L.b2t_encode_batch_dense
            _lib.check(f(tok.handle, data.ctypes.data, off.ctypes.data, len(seqs), ctypes.byref(sp), ctypes.byref(res)))
            R, W = L.b2t_result_dense_rows(res), L.b2t_result_dense_length(res)
            assert not L.b2t_result_special_tokens_mask(res) and not L.b2t_result_sequence_ids(res) and not L.b2t_result_dense_word_ids(res)
            outs.append((sp.dense_flags, bytes(np.ctypeslib.as_array(ctypes.cast(L.b2t_result_dense_ids(res), ctypes.POINTER(ctypes.c_uint8)), shape=(R * W * 4,)))))
            L.b2t_result_free(res)
        assert outs[0] == outs[1]
