"""CPU: the generated vocabularies of vocabgen.py (tokens up to 512 bytes, ids up to 2^20 - 1, shuffled merges,
ignore_merges with vocabulary-only tokens, WordPiece with other prefixes and small max_input_chars_per_word) are what they
claim, the oracle matches the reference wheel on them (and a committed fixture of the wheel's outputs where the wheel is
missing), and the soft cuts of long pre-tokens stay exact on them."""
import gzip
import hashlib
import json
import os
import numpy as np
import pytest
import helpers
import vocabgen
from vocabgen import CONFIGS, TOP_ID

from oracle import oracle as orc  # noqa: E402

BPE = [c for c in CONFIGS if c.kind == "bpe"]
N_FUZZ = 300


def char_to_byte_offsets(docs, csr):
    """char offsets of a CSR result -> byte offsets, per document"""
    offs = np.array(csr[1], dtype=np.uint32).reshape(-1, 2).copy()
    rp = csr[3]
    for d, doc in enumerate(docs):
        a, b = int(rp[d]), int(rp[d + 1])
        if a == b:
            continue
        cum = np.zeros(len(doc) + 1, dtype=np.uint32)
        np.cumsum([len(ch.encode()) for ch in doc], out=cum[1:])
        offs[a:b] = cum[offs[a:b]]
    return offs


@pytest.fixture(scope="module")
def golden():
    return json.loads(gzip.open(os.path.join(helpers.GOLDEN, "golden_vocabgen.json.gz")).read().decode("utf-8"))


@pytest.mark.parametrize("cfg", CONFIGS, ids=str)
def test_config_is_what_it_claims(cfg):
    js = json.loads(cfg.json())
    m = js["model"]
    v = m["vocab"]
    ids = sorted(v.values())
    assert len(set(ids)) == len(ids) and ids[-1] < (1 << 20)
    assert ids[-1] == (cfg.max_id if cfg.max_id is not None else len(v) - 1)
    if cfg.kind == "bpe":
        raw = [vocabgen.from_byte_level(t) for t in v]
        assert all(vocabgen.byte_level(bytes([b])) in v for b in range(256))
        assert all(a in v and b in v and a + b in v for a, b in m["merges"])
        assert vocabgen.is_monotone(v, [tuple(x) for x in m["merges"]]) == cfg.monotone
        assert max(len(r) for r in raw) == cfg.longest > 256
        if m["ignore_merges"]:   # the vocabulary-only tokens: no merge produces them
            produced = {a + b for a, b in m["merges"]}
            for t in vocabgen.vocab_only_tokens(cfg.kwargs["seed"], cfg.kwargs["vocab_only"]):
                assert vocabgen.byte_level(t) in v and vocabgen.byte_level(t) not in produced
    else:
        assert max(len(t.encode()) for t in v) == cfg.longest
        assert m["continuing_subword_prefix"] == cfg.kwargs["prefix"] and "[UNK]" in v
        if cfg.max_id == TOP_ID:
            assert v["[UNK]"] == TOP_ID


def test_generators_are_deterministic():
    """a second call gives the same tokenizer.json (no set or dict order of strings before a random draw)"""
    for cfg in CONFIGS:
        assert cfg.json() == cfg.json()


@pytest.mark.parametrize("cfg", CONFIGS, ids=str)
def test_oracle_matches_the_wheel(cfg):
    tk = helpers.wheel()
    if tk is None:
        pytest.skip("the tokenizers wheel is not importable")
    tj = cfg.json()
    docs = vocabgen.probes(cfg) + vocabgen.fuzz_docs(cfg, N_FUZZ)
    exp = helpers.wheel_csr(tk.Tokenizer.from_str(tj), docs)
    o = orc.Oracle(tj)
    helpers.assert_csr_equal(o.encode_batch(docs), exp, docs, f"{cfg} char offsets")
    if cfg.kwargs.get("pretok") != "bert":   # (byte offsets of the normalized pipeline count in the normalized text)
        got = o.encode_batch(docs, offset_type=orc.OFF_BYTE)
        helpers.assert_csr_equal(got, (exp[0], char_to_byte_offsets(docs, exp), exp[2], exp[3]), docs, f"{cfg} byte offsets")


@pytest.mark.parametrize("cfg", CONFIGS, ids=str)
def test_oracle_matches_the_pinned_fixture(cfg, golden):
    g = golden[cfg.name]
    tj = cfg.json()
    assert hashlib.sha256(tj.encode("utf-8")).hexdigest() == g["sha256"], \
        f"{cfg}: the generator's output changed; regenerate tests/golden/golden_vocabgen.json.gz with make_golden_vocabgen.py"
    docs = [c["input"] for c in g["cases"]]
    helpers.assert_csr_equal(orc.Oracle(tj).encode_batch(docs), helpers.cases_to_csr(g["cases"]), docs, f"{cfg} fixture")


def long_pretokens(cfg):
    """raw bytes of every pre-token of more than 256 bytes of the targeted documents: under the configuration's own
    pre-tokenizer, and each whole document (what no-regex ByteLevel makes of it)"""
    o = orc.Oracle(cfg.json())
    out = []
    for d in vocabgen.bpe_probes(cfg):
        b = d.encode()
        out += [b[s:e] for s, e in o.pre_tokenize(d) if e - s > 256]
        if len(b) > 256:
            out.append(b)
    return sorted(set(out))


@pytest.mark.parametrize("cfg", BPE, ids=str)
def test_soft_cuts_are_exact(cfg):
    """merging a long pre-token whole gives the tokens of its soft-cut pieces merged one by one (ignore_merges off for
    the pieces: they get no whole-word lookup), unless the whole pre-token is a vocabulary entry itself"""
    tk = helpers.wheel()
    if tk is None:
        pytest.skip("the tokenizers wheel is not importable")
    js = json.loads(cfg.json())
    vocab = js["model"]["vocab"]
    tokens = [vocabgen.from_byte_level(t) for t in vocab]
    whole_model = tk.Tokenizer.from_str(json.dumps(js)).model
    js["model"]["ignore_merges"] = False
    piece_model = tk.Tokenizer.from_str(json.dumps(js)).model
    n_cut = 0
    for raw in long_pretokens(cfg):
        if vocabgen.byte_level(raw) in vocab:
            continue
        pieces = vocabgen.soft_cuts(tokens, raw)
        assert b"".join(pieces) == raw
        n_cut += len(pieces) > 1
        whole = [t.id for t in whole_model.tokenize(vocabgen.byte_level(raw))]
        parts = [t.id for p in pieces for t in piece_model.tokenize(vocabgen.byte_level(p))]
        assert whole == parts, (cfg.name, raw[:80], [len(p) for p in pieces][:20])
    assert n_cut > 0
    # runs of a chain letter are never cut (every pair and triple of them is inside a token): K2L merges them whole
    assert vocabgen.soft_cuts(tokens, b"a" * 2100) == [b"a" * 2100]
    # the piece construction: cut around every "!" into copies of the vocabulary-only token
    if vocabgen.byte_level(vocabgen.PIECE_TOKEN) in vocab:
        pieces = vocabgen.soft_cuts(tokens, vocabgen.PIECE_RUN.encode())
        assert pieces[0] == vocabgen.PIECE_TOKEN.encode() and pieces[1] == b"!" and len(pieces) == 121


def test_piece_token_comes_out_as_bytes():
    """under ignore_merges and no regex, the run of PIECE_TOKEN pieces is one pre-token that is not in the vocabulary:
    the reference merges it (into bytes: no merge touches its letters), and never returns the vocabulary-only id for a
    piece of it; the piece alone is a whole word"""
    tk = helpers.wheel()
    cfg = vocabgen.BY_NAME["bpe_noregex_ignore"]
    tj = cfg.json()
    piece_id = json.loads(tj)["model"]["vocab"][vocabgen.PIECE_TOKEN]
    for enc in ([tk.Tokenizer.from_str(tj)] if tk else []) + [None]:
        if enc is None:
            ids = orc.Oracle(tj).encode_batch([vocabgen.PIECE_RUN, vocabgen.PIECE_TOKEN])
            run, alone = ids[0][:int(ids[3][1])], ids[0][int(ids[3][1]):]
        else:
            run, alone = (e.ids for e in enc.encode_batch([vocabgen.PIECE_RUN, vocabgen.PIECE_TOKEN], add_special_tokens=False))
        assert len(run) == len(vocabgen.PIECE_RUN) and piece_id not in list(run)
        assert list(alone) == [piece_id]
