"""GPU (-m gpu): the engine against the oracle on the generated vocabularies of vocabgen.py -- tokens up to 512 bytes, ids
up to 2^20 - 1, shuffled (non-monotone) merges, ignore_merges with vocabulary-only tokens of up to 300 bytes, WordPiece
with the prefixes "##", "", "▁" and "@@" and max_input_chars_per_word of 1 to 104 -- bit for bit: ids, char and byte
offsets, word ids and row_ptr, word cache on and off, ids only, and the device-resident entry point.  Long probes start
at page offsets 0, 1 and 2047, so a 256-byte token ends at the far end of the BPE halo and a 104-character WordPiece word
of 4-byte letters fills the 416-byte one.  Each test first asserts, from the expected output, that its documents reach
what they are there for.  Also: ids of 2^20 refused, added tokens with ids just below 2^20 extracted on the device, and
dense rows of high ids."""
import json
import numpy as np
import pytest
import helpers
import vocabgen
from vocabgen import CONFIGS, TOP_ID

pytestmark = pytest.mark.gpu

from tokenizers_b200 import Tokenizer, _lib  # noqa: E402
from tokenizers_b200.tokenizer import UnsupportedConfig  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from helpers import PAGE, place  # noqa: E402

LONG_STARTS = [0, 1, 2047]   # page offsets of a long probe's first byte
N_FUZZ = 400


def long_slots(probes):
    """each probe, a document of its own, with its first byte at each of LONG_STARTS"""
    slots, k = [], 1
    for p in probes:
        for d in LONG_STARTS:
            slots.append((p, k * PAGE + d, "start"))
            k += 2 + len(p.encode()) // PAGE
    return slots


_batches = {}


def batch(cfg):
    """-> (tokenizer.json, docs, expected char-offset CSR): the configuration's targeted documents (those over 16 bytes
    placed at LONG_STARTS) and fuzz documents"""
    if cfg.name not in _batches:
        tj = cfg.json()
        pr = vocabgen.probes(cfg)
        docs = place(long_slots([p for p in pr if len(p.encode()) > 16]), "doc") + [p for p in pr if len(p.encode()) <= 16]
        docs += vocabgen.fuzz_docs(cfg, N_FUZZ)
        _batches[cfg.name] = (tj, docs, orc.Oracle(tj).encode_batch(docs))
    return _batches[cfg.name]


def token_bytes(tj):
    """id -> length in bytes of its token"""
    v = json.loads(tj)["model"]["vocab"]
    if json.loads(tj)["model"]["type"] == "BPE":
        return {i: len(vocabgen.from_byte_level(t)) for t, i in v.items()}
    return {i: len(t.encode()) for t, i in v.items()}


def assert_reached(cfg, tj, docs, exp):
    """the premises of the comparison, from the expected output"""
    ids = exp[0]
    js = json.loads(tj)
    v = js["model"]["vocab"]
    if cfg.max_id == TOP_ID:
        assert np.any(ids == TOP_ID), f"{cfg}: id 2^20 - 1 never occurs"
    assert ids.max() >= (1 << 17) or cfg.max_id is None
    if cfg.kind == "bpe":
        tb = token_bytes(tj)
        lens = np.array([tb[int(i)] for i in ids])
        assert np.any((lens > 32) & (lens <= 256)), f"{cfg}: no token of 33..256 bytes"
        assert np.any(lens > 256), f"{cfg}: no token of more than 256 bytes"
        if js["model"]["ignore_merges"]:
            only = {v[vocabgen.byte_level(t)]: len(t) for t in vocabgen.vocab_only_tokens(cfg.kwargs["seed"], cfg.kwargs["vocab_only"])}
            seen = {only[int(i)] for i in ids if int(i) in only}
            assert any(46 < n <= 256 for n in seen), f"{cfg}: no vocabulary-only token of 47..256 bytes (page-kernel whole word)"
            assert any(n > 256 for n in seen), f"{cfg}: no vocabulary-only token of more than 256 bytes (K2L whole word)"
            if cfg.kwargs.get("pretok") == "noregex":   # pieces of one long pre-token get no whole-word lookup
                piece = v[vocabgen.PIECE_TOKEN]
                rp = exp[3]
                d = docs.index(vocabgen.PIECE_RUN)
                run = ids[int(rp[d]):int(rp[d + 1])]
                assert len(run) == len(vocabgen.PIECE_RUN) and piece not in run, "the piece must come out as bytes"
                assert piece in ids, "the piece token alone is a whole word"
    else:
        unk = v["[UNK]"]
        m = cfg.kwargs["max_chars"]
        o = orc.Oracle(tj)
        too_long, failed = vocabgen.abc_word(m + 1), "ab" + vocabgen.WP_MISSING
        assert too_long in docs and failed in docs
        assert list(o.encode_batch([too_long, failed])[0]) == [unk, unk], f"{cfg}: [UNK] from the length limit and from a failed match"
        assert unk not in o.encode_batch([too_long[:m]])[0]
        assert np.any(ids == unk)


@pytest.mark.parametrize("cfg", CONFIGS, ids=str)
def test_generated_vocabulary(cfg):
    """ids, char and byte offsets, word ids, row_ptr with the word cache on and off; ids only; the device-resident entry"""
    tj, docs, exp = batch(cfg)
    assert_reached(cfg, tj, docs, exp)
    bert = cfg.kwargs.get("pretok") == "bert"   # (byte offsets are refused behind the normalizer)
    helpers.check(tj, docs, cfg.name, byte_offsets=not bert)
    data, off = helpers.pack_docs(docs)
    tok = Tokenizer.from_str(tj)
    be = tok.encode_batch_csr(data, off, offsets=False, word_ids=False)
    assert be.offsets is None and be.word_ids is None
    helpers.assert_csr_equal((be.ids, None, None, be.row_ptr), exp, docs, f"{cfg} ids only")
    got = helpers.device_csr(tok, data, off, _lib.WANT_OFFSETS | _lib.WANT_WORD_IDS)
    helpers.assert_csr_equal(got, exp, docs, f"{cfg} device entry point")


def test_ids_of_2_pow_20_are_refused():
    """a vocabulary id of 2^20 does not fit the page kernel's 20 id bits: the engine refuses the vocabulary
    (B2T_ERR_UNSUPPORTED, raised by the tokenizer as UnsupportedConfig); 2^20 - 1 is accepted"""
    js = json.loads(vocabgen.BY_NAME["bpe_noregex_high"].json())
    v = js["model"]["vocab"]
    top = next(t for t, i in v.items() if i == TOP_ID)
    Tokenizer.from_str(json.dumps(js))
    v[top] = 1 << 20
    with pytest.raises(UnsupportedConfig, match="2\\^20"):
        Tokenizer.from_str(json.dumps(js))
    wp = json.loads(vocabgen.BY_NAME["wp_empty_5"].json())
    wp["model"]["vocab"]["[UNK]"] = 1 << 20
    with pytest.raises(UnsupportedConfig, match="2\\^20"):
        Tokenizer.from_str(json.dumps(wp))


def added_json(cfg_name, ids):
    """the configuration with ADDED_TOKEN_SPECS (those not in its vocabulary) as added tokens of the given ids"""
    js = json.loads(vocabgen.BY_NAME[cfg_name].json())
    v = js["model"]["vocab"]
    specs = [s for s in helpers.ADDED_TOKEN_SPECS if vocabgen.byte_level(s[0]) not in v]
    js["added_tokens"] = [{"id": i, "content": c, "single_word": sw, "lstrip": ls, "rstrip": rs, "normalized": nm, "special": sp}
                          for i, (c, sw, ls, rs, nm, sp) in zip(ids, specs)]
    return json.dumps(js), len(specs)


def test_added_token_of_id_2_pow_20_is_not_extracted_on_the_device():
    """b2t_engine_set_added_tokens refuses an added id of 2^20 (B2T_ERR_UNSUPPORTED); the tokenizer then splits the added
    tokens on the host, where the id needs no packing, and still gives the reference's output.  2^20 - 1 is accepted."""
    for top, dev in ((TOP_ID, True), (1 << 20, False)):
        tj, n = added_json("bpe_gpt2", [top - k for k in range(20)])
        tok = Tokenizer.from_str(tj)
        assert tok._dev_added == dev
        docs = helpers.added_token_docs(7, 200)
        got = tok.encode_batch(docs, add_special_tokens=False)
        ref = helpers.oracle_backed_tokenizer(tj).encode_batch(docs, add_special_tokens=False)
        assert [list(e.ids) for e in got] == [list(e.ids) for e in ref]
        assert any(top in list(e.ids) for e in ref)
    L = _lib.lib()
    for i, rc in ((TOP_ID, _lib.B2T_OK), (1 << 20, _lib.B2T_ERR_UNSUPPORTED)):
        b = np.frombuffer(b"<x>", dtype=np.uint8).copy()
        o = np.array([0, 3], dtype=np.uint32)
        ids = np.array([i], dtype=np.uint32)
        fl = np.zeros(1, dtype=np.uint8)
        assert L.b2t_engine_set_added_tokens(tok.handle, 1, b.ctypes.data, o.ctypes.data, ids.ctypes.data, fl.ctypes.data) == rc


@pytest.mark.parametrize("byte_offsets", [False, True])
def test_added_tokens_with_high_ids_on_the_device(byte_offsets):
    """device extraction (FLAG_ADDED_IDS) of added tokens with ids just below 2^20, in front of a vocabulary of ids just
    below them: bit 31 marks the added ids and must survive next to 20-bit ids"""
    used = set(json.loads(vocabgen.BY_NAME["bpe_noregex_high"].json())["model"]["vocab"].values())
    free = [i for i in range(TOP_ID, TOP_ID - 100, -1) if i not in used][:20]   # interleaved with the vocabulary's ids
    tj, n = added_json("bpe_noregex_high", free)
    tj = json.loads(tj)
    tj["pre_tokenizer"] = vocabgen.PRETOKENIZERS["gpt2"]
    tj = json.dumps(tj)
    tok, ref = Tokenizer.from_str(tj), helpers.oracle_backed_tokenizer(tj)
    assert tok._dev_added
    docs = helpers.added_token_docs(8, 1500) + vocabgen.bpe_probes(vocabgen.BY_NAME["bpe_noregex_high"])
    data, off = helpers.pack_docs(docs)
    exp = helpers.host_added_csr(ref, data, off, byte_offsets)
    marked = exp[0][exp[0] >> 31 != 0] & np.uint32(0x7FFFFFFF)
    assert marked.size > 0 and marked.min() >= TOP_ID - 100
    assert np.any((exp[0] >> 31 == 0) & (exp[0] == TOP_ID))
    got = tok._engine_rows(data, off, _lib.WANT_OFFSETS | _lib.WANT_WORD_IDS | _lib.FLAG_ADDED_IDS | (_lib.OFFSETS_BYTES if byte_offsets else 0))
    helpers.assert_csr_equal(got, exp, docs, f"added high ids bytes={byte_offsets}")


@pytest.mark.parametrize("length", [48, None])
def test_dense_rows_with_high_ids(length):
    """b2t_encode_batch_dense with ids up to 2^20 - 1 (and that pad id): a fixed length and BatchLongest"""
    cfg = vocabgen.BY_NAME["bpe_llama3_ignore"]
    tj, docs, exp = batch(cfg)
    data, off = helpers.pack_docs(docs)
    max_length = 48 if length else 4096
    tok = Tokenizer.from_str(tj)
    tok.enable_truncation(max_length)
    tok.enable_padding(length=length, pad_id=TOP_ID)
    got = tok.encode_batch_dense(data, off, add_special_tokens=False)
    want = orc.dense_rows(exp[0], exp[3], length=length or 0, pad_to_multiple_of=0, max_length=max_length, pad_id=TOP_ID,
                          truncate_left=False, pad_left=False, pre=[], post=[])
    assert np.any(want[0][want[1] == 1] == TOP_ID)
    assert np.array_equal(got["input_ids"], want[0]) and np.array_equal(got["attention_mask"], want[1]) and np.array_equal(got["lengths"], want[2])
