"""The PreTokenizer seam (b2t_pre_tokenize_batch, Tokenizer.pre_tokenize_batch) against the oracle: the only entry point
that returns what the scan kernels K1 compute -- the split bitmap and the removed-whitespace bitmap -- before the model
kernel K2 can hide a mistake behind a merge.

The seam splits the text as given: neither the engine's BertNormalizer nor its added tokens apply, as with the
reference's `pre_tokenizer.pre_tokenize_str`.  Every pre-tokenizer kind runs here, and the engine features the seam has
to ignore: fuzz and corpus documents, edge batches, probes at page edges and at the 2 MiB scan-block edge, and 50 MiB
tiled batches where every K1 warp owns several pages (GPU, -m gpu); the oracle's splits against the wheel's (CPU)."""
import ctypes
import json
import random
import numpy as np
import pytest
import helpers, fuzzgen, corpus

from tokenizers_b200 import Tokenizer, _lib  # noqa: E402
from oracle import oracle as orc  # noqa: E402

tk = helpers.wheel()

PIPELINES = ["gpt2_style", "gpt2_noregex", "gpt2_prefix", "llama3_style", "wordpiece", "bert_pretok", "bert_uncased",
             "added_gpt2_style", "added_wordpiece"]
BYTE_LEVEL = ["gpt2_style", "gpt2_noregex", "gpt2_prefix", "llama3_style", "added_gpt2_style"]
BERT = ["bert_pretok", "bert_uncased"]
DROPS_WHITESPACE = ["wordpiece", "added_wordpiece"] + BERT   # Whitespace and BertPreTokenizer remove whitespace
HOST_BYTES = 50 << 20


def pipeline_json(name):
    """helpers.pipeline_json, and bert_pretok: WordPiece behind BertPreTokenizer without a normalizer"""
    if name == "bert_pretok":
        js = json.loads(helpers.asset_json("wordpiece"))
        js["pre_tokenizer"] = {"type": "BertPreTokenizer"}
        return json.dumps(js)
    return helpers.pipeline_json(name)


_engines = {}


def engine(name):
    if name not in _engines:
        tj = pipeline_json(name)
        _engines[name] = (Tokenizer.from_str(tj), orc.Oracle(tj))
    return _engines[name]


def seam(tok, data, doc_off):
    """b2t_pre_tokenize_batch through the C ABI -> (offsets u32[K, 2], row_ptr u64[n + 1])"""
    data = np.ascontiguousarray(data, dtype=np.uint8)
    doc_off = np.ascontiguousarray(doc_off, dtype=np.uint64)
    n = len(doc_off) - 1
    L = _lib.lib()
    res = ctypes.c_void_p()
    _lib.check(L.b2t_pre_tokenize_batch(tok.handle, data.ctypes.data if data.size else None, doc_off.ctypes.data, n, ctypes.byref(res)))
    try:
        assert L.b2t_result_on_device(res) == 0 and L.b2t_result_n_docs(res) == n
        assert not L.b2t_result_ids(res) and not L.b2t_result_word_ids(res)
        K = L.b2t_result_n_tokens(res)

        def view(ptr, count, dtype):
            if count == 0:
                return np.zeros(0, dtype=dtype)
            return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint8)), shape=(count * np.dtype(dtype).itemsize,)).view(dtype).copy()
        return view(L.b2t_result_offsets(res), 2 * K, np.uint32).reshape(-1, 2), view(L.b2t_result_row_ptr(res), n + 1, np.uint64)
    finally:
        L.b2t_result_free(res)


def oracle_seam(o, data, doc_off):
    """Oracle.pre_tokenize per document, in the form of helpers.tiled_expectation's pieces: (None, offsets, None, row_ptr)"""
    raw = np.ascontiguousarray(data, dtype=np.uint8).tobytes()
    doc_off = np.asarray(doc_off, dtype=np.uint64)
    parts = [o.pre_tokenize_bytes(raw[int(a):int(b)]) for a, b in zip(doc_off[:-1], doc_off[1:])]
    rp = np.zeros(len(parts) + 1, dtype=np.uint64)
    if parts:
        np.cumsum([len(p) for p in parts], out=rp[1:])
    offs = np.concatenate(parts) if parts else np.zeros((0, 2), dtype=np.uint32)
    return None, offs.astype(np.uint32).reshape(-1, 2), None, rp


def assert_seam_equal(got, exp, data, doc_off, what):
    """offsets and row_ptr equal; otherwise the message names the first document whose splits differ"""
    go, grp = np.asarray(got[0], dtype=np.uint32).reshape(-1, 2), np.asarray(got[1], dtype=np.uint64)
    eo, erp = np.asarray(exp[1], dtype=np.uint32).reshape(-1, 2), np.asarray(exp[3], dtype=np.uint64)
    if np.array_equal(grp, erp) and np.array_equal(go, eo):
        return
    n = len(doc_off) - 1
    assert len(grp) == n + 1, f"{what}: row_ptr of {len(grp)} entries for {n} documents"
    counts_differ = np.nonzero(np.diff(grp.astype(np.int64)) != np.diff(erp.astype(np.int64)))[0]
    d = int(counts_differ[0]) if counts_differ.size else n
    upto = int(erp[d]) if d < n else len(eo)   # before document d the rows line up
    k = min(upto, len(go), len(eo))
    pair_differ = np.nonzero((go[:k] != eo[:k]).any(axis=1))[0]
    if pair_differ.size:
        d = min(d, int(np.searchsorted(erp.astype(np.int64), int(pair_differ[0]), side="right")) - 1)
    if d >= n:
        raise AssertionError(f"{what}: {len(go)} splits, expected {len(eo)}")
    raw = np.asarray(data, dtype=np.uint8)[int(doc_off[d]):int(doc_off[d + 1])].tobytes()
    text = raw.decode("utf-8", "replace")
    raise AssertionError(f"{what}: first differing document {d} of {n} (batch bytes {int(doc_off[d])}..{int(doc_off[d + 1])}): "
                         f"{text[:300]!r}{'...' if len(text) > 300 else ''}\n"
                         f"  expected {eo[int(erp[d]):int(erp[d + 1])][:40].tolist()}\n  got      {go[int(grp[d]):int(grp[d + 1])][:40].tolist()}")


def check_docs(name, docs, what):
    tok, o = engine(name)
    data, off = helpers.pack_docs(docs)
    got = seam(tok, data, off)
    assert_seam_equal(got, oracle_seam(o, data, off), data, off, f"{name} {what}")
    return got


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------ documents
def fuzz_and_corpus_batches():
    rng = random.Random(7)
    out = [("fuzz short", fuzzgen.rand_docs(601, 2000, max_len=40)),
           ("fuzz long", fuzzgen.rand_docs(602, 800, max_len=300)),
           ("long runs", [fuzzgen.run_doc(rng) for _ in range(600)])]   # across 32 B chunks and the Llama-3 window
    for kind in (1, 2, 4, 5):
        data, off = corpus.generate(kind, 610 + kind, 0, 1500)
        out.append((f"corpus {kind}", corpus.to_strings(data, off)))
    return out


WHITESPACE_ONLY = [" ", "  ", "\n", "\t \r\n", " " * 40, "\xa0", "\u3000", "\u2003 \u2009", "\x0b\x0c", "\n" * 33]
RUNS = ["a", " ", "\n", "1", "!", "\u00e9", "\u4e2d", "ab "]


def edge_batches():
    """no documents, empty documents, whitespace only, one byte, and single runs of 2047 / 2048 / 2049 bytes (the batch
    ends on either side of the first page edge), each alone and all in one batch"""
    out = [("no documents", []), ("empty documents", ["", "", ""]), ("whitespace only", WHITESPACE_ONLY),
           ("one byte", ["x"]), ("one space", [" "]), ("empty and one byte", ["", "x", ""])]
    runs = []
    for n in (2047, 2048, 2049):
        for r in RUNS:
            b = (r.encode() * n)[:n]
            while True:   # (whole characters only: cut a multi-byte run short and pad it with ASCII)
                try:
                    s = b.decode()
                    break
                except UnicodeDecodeError:
                    b = b[:-1]
            runs.append(s + "x" * (n - len(s.encode())))
    out += [(f"run of {len(s.encode())} bytes ({s[:2]!r}...)", [s]) for s in runs]
    out.append(("all runs", runs))
    return out


def probes_for(name):
    """page-edge probes: the BPE ones for ByteLevel; WordPiece words for Whitespace and Bert, and for Bert the characters
    a BertNormalizer would expand -> [(probes, deltas)]"""
    if name in BYTE_LEVEL:
        return [(helpers.bpe_probes(), helpers.DELTAS)]
    out = [(helpers.wordpiece_probes(100), helpers.DELTAS)]
    if name in BERT:
        out.append((helpers.BERT_PROBES, [-9, -3, -2, -1, 0, 1, 2, 3, 9]))
    return out


# ------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", PIPELINES)
def test_fuzz_corpus_and_edge_batches(name):
    for what, docs in fuzz_and_corpus_batches() + edge_batches():
        got = check_docs(name, docs, what)
        if what == "whitespace only" and name in DROPS_WHITESPACE:
            assert got[0].shape[0] == 0 and not got[1].any(), f"{name}: splits in whitespace-only documents"
        if what == "no documents":
            assert got[0].shape[0] == 0 and got[1].tolist() == [0]


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["doc", "text"])
@pytest.mark.parametrize("name", PIPELINES)
def test_probes_at_page_edges(name, form):
    for probes, deltas in probes_for(name):
        check_docs(name, helpers.place(helpers.page_slots(probes, deltas), form), f"page edges {form} ({len(probes)} probes)")


@pytest.mark.gpu
@pytest.mark.parametrize("name", PIPELINES)
def test_probes_at_the_scan_block_edge(name):
    probes = [p for ps, _ in probes_for(name) for p in ps]
    sel = [probes[i] for i in range(0, len(probes), max(1, len(probes) // 8))][:8]
    for form in ("doc", "text"):
        check_docs(name, helpers.place(helpers.scan_block_slots(sel), form), f"2 MiB {form}")


def tiled(name):
    base = helpers.scale_base(name if name != "bert_pretok" else "wordpiece", seed=11)
    data, off, shims = helpers.tiled_batch(*base, HOST_BYTES, seed=12)
    return base, data, off, shims


def assert_kb(name, n_scanned):
    """the regime of the scale tests: K1 warps of 4 KB or more (Llama-3 at its own occupancy)"""
    kb = helpers.k1_kb(n_scanned, sm_count(), name == "llama3_style")
    assert kb >= 4, f"{n_scanned} scanned bytes give {kb} KB per K1 warp on {sm_count()} SMs; the test needs >= 4"
    print(f"{name}: {n_scanned / 2**20:.1f} MiB scanned, kb = {kb}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", PIPELINES)
def test_multi_page_warp_ranges(name):
    """50 MiB tiled batches, compared in full: the bytes K1 scans are the input's (plus the prefix spaces of
    gpt2_prefix, so the input's size is the bound used), under bert_uncased too"""
    tok, o = engine(name)
    base, data, off, shims = tiled(name)
    assert_kb(name, int(data.size))
    got = seam(tok, data, off)
    exp = helpers.tiled_expectation(lambda d, f: oracle_seam(o, d, f), *base, shims)
    assert_seam_equal(got, exp, data, off, f"{name} {data.size} bytes")


@pytest.mark.gpu
@pytest.mark.parametrize("name", [p for p in PIPELINES if p != "bert_uncased" and not p.startswith("added_")])
def test_seam_split_counts_equal_word_counts(name):
    """each document's split count from the seam equals max(word id) + 1 of the encode path (0 without tokens): K1's split
    bitmap against the word ids K2 emits, on the batches of test_multi_page_warp_ranges, without the oracle"""
    tok, _ = engine(name)
    _, data, off, _ = tiled(name)
    _, rp = seam(tok, data, off)
    be = tok.encode_batch_csr(data, off)
    erp, wid = np.asarray(be.row_ptr, dtype=np.int64), np.asarray(be.word_ids, dtype=np.int64)
    words = np.zeros(len(off) - 1, dtype=np.int64)
    has = np.nonzero(np.diff(erp) > 0)[0]
    if has.size:
        words[has] = np.maximum.reduceat(wid, erp[has]) + 1
    splits = np.diff(rp.astype(np.int64))
    bad = np.nonzero(splits != words)[0]
    if bad.size:
        d = int(bad[0])
        raise AssertionError(f"{name}: document {d} has {splits[d]} splits and {words[d]} words "
                             f"({len(bad)} documents differ): {data[int(off[d]):int(off[d + 1])].tobytes()[:300]!r}")


# the documents on which normalizing before the split moved the seam's offsets: accents, upper case, CJK, characters
# clean_text removes or turns into spaces
NORMALIZER_DOCS = ["H\u00e9llo w\u00f6rld \u4e2d\u6587\u0301\u0301 x", "\u00c0\u00c9\u00ce\u00d5\u00dc \u00e0\u00e9\u00ee\u00f5\u00fc Stra\u00dfe",
                   "HELLO World \u0130stanbul \u01c5emal", "\u4e2d\u6587\u5b57 \u65e5\u672c\u8a9e\u306e\u6587 \ud55c\uad6d\uc5b4",
                   "a\x00b\x01c d\ufffde f\x7fg", "tab\there\x0bvt\x0cff\x85nel", "zero\u200bwidth\u200d joiner\ufeffbom",
                   "na\u00efve cafe\u0301 re\u0301sume\u0301", "x\u4e2dy\u6587z", "\u0301leading mark", "trailing mark\u0301", "!?...,;:\u00bf\u00a1"]
REFUSED_RUN = "a\u08d4\u0316x"   # a mark strip_accents keeps next to another mark: N1 refuses it (test_bert_alignment.TABLE)


@pytest.mark.gpu
def test_seam_ignores_the_normalizer():
    """under bert_uncased the seam splits the raw text, like the wheel's pre_tokenize_str; encode still normalizes"""
    name = "bert_uncased"
    tok, o = engine(name)
    # (normalized, the CJK characters would be split apart and every offset after the first accent would move)
    assert check_docs(name, [NORMALIZER_DOCS[0]], "accents, CJK and marks")[0].tolist() == [[0, 6], [7, 13], [14, 24], [25, 26]]
    marks = ["\u0301"] * 2000   # every document vanishes under normalization
    long_marks = ["".join(chr(0x300 + (i % 0x30)) for i in range(20000))]
    for what, docs in (("normalizer-sensitive", NORMALIZER_DOCS), ("2000 single marks", marks), ("20000 marks", long_marks),
                       ("all", NORMALIZER_DOCS + marks + long_marks)):
        got = check_docs(name, docs, what)
        if docs is marks:
            assert np.diff(got[1].astype(np.int64)).tolist() == [1] * len(marks)
        data, off = helpers.pack_docs(docs)
        be = tok.encode_batch_csr(data, off)   # the encode path: the normalized text, offsets into the original
        helpers.assert_csr_equal((be.ids, be.offsets, be.word_ids, be.row_ptr), o.encode_batch_csr(data, off), docs, f"encode {what}")
    # the refused run: the seam splits it (no normalization runs), encode still refuses it
    for docs in ([REFUSED_RUN], ["fine", REFUSED_RUN, "also fine"]):
        check_docs(name, docs, "refused run")
        with pytest.raises(_lib.B2TError) as ei:
            tok.encode_batch_csr(*helpers.pack_docs(docs))
        assert ei.value.code == _lib.B2T_ERR_UNSUPPORTED and "combining character" in str(ei.value)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["added_gpt2_style", "added_wordpiece"])
def test_seam_ignores_added_tokens(name):
    """documents full of the engine's added tokens: the seam splits them as plain text (<|endoftext|> into several splits)"""
    tok, o = engine(name)
    docs = helpers.added_token_docs(31, 400)
    got = check_docs(name, docs, "added-token documents")
    i = docs.index("<|endoftext|>")
    assert len(o.pre_tokenize("<|endoftext|>")) > 1 and got[1][i + 1] - got[1][i] == len(o.pre_tokenize("<|endoftext|>"))


# ------------------------------------------------------------------------------------------ CPU
def wheel_splits(pt, doc):
    """the wheel's pre_tokenize_str offsets (characters of the original) in bytes"""
    cum = np.concatenate([[0], np.cumsum([len(c.encode("utf-8")) for c in doc])])
    return [(int(cum[a]), int(cum[b])) for _, (a, b) in pt.pre_tokenize_str(doc)]


@pytest.mark.skipif(tk is None, reason="reference wheel not importable")
@pytest.mark.parametrize("name", PIPELINES)
def test_oracle_splits_match_the_wheel(name):
    """Oracle.pre_tokenize, the expectation of every GPU test above, against the reference's pre-tokenizer itself: the
    text as given, without the normalizer or the added tokens"""
    tj = pipeline_json(name)
    pt, o = tk.Tokenizer.from_str(tj).pre_tokenizer, orc.Oracle(tj)
    batches = fuzz_and_corpus_batches() + [("edges", [d for _, ds in edge_batches() for d in ds]),
                                           ("normalizer-sensitive", NORMALIZER_DOCS + ["\u0301", "\u0301" * 50, REFUSED_RUN]),
                                           ("added tokens", helpers.added_token_docs(31, 400))]
    for what, docs in batches:
        for d in docs:
            assert o.pre_tokenize(d) == wheel_splits(pt, d), f"{name} {what}: {d!r}"
