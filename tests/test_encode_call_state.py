"""An encode call keeps what belongs to it (zero_copy, the engine result its arrays are views of) out of the Tokenizer,
so that one Tokenizer serves calls from several host threads at once."""
import json, threading
import numpy as np
import pytest
import helpers

FIELDS = ("ids", "offsets", "word_ids", "row_ptr", "type_ids", "special_tokens_mask")


def _tokenizer_json():
    """gpt2_style with the added tokens of helpers, offset trimming and a special-token template (single and pair)"""
    js = json.loads(helpers.with_added_tokens(helpers.asset_json("gpt2_style"), template=True))
    js["post_processor"] = {"type": "Sequence", "processors": [
        {"type": "ByteLevel", "add_prefix_space": True, "trim_offsets": True, "use_regex": True}, js["post_processor"]]}
    return json.dumps(js)


def _assert_same(got, exp, what):
    for f in FIELDS:
        g, e = getattr(got, f), getattr(exp, f)
        assert (g is None) == (e is None) and (g is None or np.array_equal(g, e)), f"{what}: {f} differ"


def test_encode_calls_write_no_tokenizer_state():
    tok = helpers.oracle_backed_tokenizer(_tokenizer_json())
    docs = helpers.added_token_docs(3, 60)
    data, off = helpers.pack_docs(docs)
    [e.tokens for e in tok.encode_batch(docs)]  # warm-up: fills the lazy caches (trim tables, reverse vocabulary)
    writes = []

    class Watched(type(tok)):
        def __setattr__(self, name, value):
            writes.append(name)
            super().__setattr__(name, value)
    tok.__class__ = Watched
    snapshot = dict(vars(tok))
    copied = tok.encode_batch_csr(data, off, add_special_tokens=True)
    _assert_same(tok.encode_batch_csr(data, off, add_special_tokens=True, zero_copy=True), copied, "zero_copy")
    tok.encode_batch(docs)
    tok.encode_batch_fast(docs)
    tok.encode(docs[5], docs[6])
    assert writes == []
    assert vars(tok).keys() == snapshot.keys() and all(vars(tok)[k] is v for k, v in snapshot.items())


@pytest.mark.gpu
def test_threads_share_one_tokenizer():
    """One thread keeps zero-copy views, the other takes copies, four rounds each started together; once both have
    finished, every result still equals the one computed before, one call at a time."""
    from tokenizers_b200 import Tokenizer
    tok = Tokenizer.from_str(_tokenizer_json())
    batches = [helpers.pack_docs(helpers.added_token_docs(20 + i, 6000)) for i in range(2)]
    exp = [tok.encode_batch_csr(*b) for b in batches]
    barrier = threading.Barrier(2, timeout=300)
    got, errs = ([], []), []

    def work(i):
        try:
            for _ in range(4):
                barrier.wait()
                got[i].append(tok.encode_batch_csr(*batches[i], zero_copy=(i == 0)))
        except Exception as ex:  # pragma: no cover
            barrier.abort()
            errs.append(ex)
    ts = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    [t.start() for t in ts]; [t.join() for t in ts]
    assert not errs, errs
    for i in range(2):
        assert len(got[i]) == 4
        for r, be in enumerate(got[i]):
            _assert_same(be, exp[i], f"thread {i} round {r}")
    # the views keep their engine result alive, and with it the engine, which must outlive its results
    assert all(be._owner is not None and be._owner._tok is tok for be in got[0])
