"""GPU (-m gpu): full parity on batches large enough that every warp of the pre-tokenization scan (K1) owns several pages.

Up to about 33 MiB (16.5 MiB for Llama-3) on a 132-SM H100 a K1 warp owns 2 KB, one page; only above that does a warp
carry its state (the class carry, the GPT-2 overflow chain, the stage-B state, the half-page sums, the added-token words)
from one page to the next.  The batches here are tiled (helpers.tiled_batch): copies of a base set of documents behind
shims of varying length, so the expected output comes from the oracle on the base set and compares in full."""
import numpy as np
import pytest
import helpers

pytestmark = pytest.mark.gpu

from tokenizers_b200 import Tokenizer, _lib  # noqa: E402
from oracle import oracle as orc  # noqa: E402

HOST_BYTES = 50 << 20     # one chunk of the host path (64 MiB)
DEVICE_BYTES = 116 << 20  # b2t_encode_batch_device does not chunk
ALL = _lib.WANT_OFFSETS | _lib.WANT_WORD_IDS


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def assert_kb(n_scanned, llama3, at_least):
    """the regime this test is for: K1 warps of `at_least` KB or more (see launch_pretok)"""
    kb = helpers.k1_kb(n_scanned, sm_count(), llama3)
    assert kb >= at_least, f"{n_scanned} scanned bytes give {kb} KB per K1 warp on {sm_count()} SMs; the test needs >= {at_least}"
    print(f"{n_scanned / 2**20:.1f} MiB scanned, kb = {kb}")
    return kb


def scanned_bytes(name, data, off, base, shims):
    """bytes the K1 scan sees: the batch after the BertNormalizer (with add_prefix_space a few more than the input,
    which is the bound used)"""
    n = int(data.size)
    if name == "bert_uncased":
        nz = orc.BertNormalizer(**helpers.BERT_UNCASED)
        bd, bo = base
        raw = bd.tobytes()
        norm = sum(len(nz.normalize(raw[int(bo[d]):int(bo[d + 1])])[0]) for d in range(len(bo) - 1))
        n = len(shims) * norm + sum(shims)   # (the shims are lower-case ASCII)
    return n


_o = {}


def oracle(tj):
    if tj not in _o:
        _o[tj] = orc.Oracle(tj)
    return _o[tj]


@pytest.mark.parametrize("name", ["gpt2_style", "gpt2_noregex", "gpt2_prefix", "llama3_style", "wordpiece", "bert_uncased"])
def test_host_path_multi_page_warps(name):
    tj = helpers.pipeline_json(name)
    tok, o = Tokenizer.from_str(tj), oracle(tj)
    base = helpers.scale_base(name, seed=3)
    data, off, shims = helpers.tiled_batch(*base, HOST_BYTES, seed=4)
    assert data.size < 64 << 20, "one chunk of the host path"
    assert_kb(scanned_bytes(name, data, off, base, shims), name == "llama3_style", 4)
    exp = helpers.tiled_expectation(o.encode_batch_csr, *base, shims)
    be = tok.encode_batch_csr(data, off)
    helpers.assert_csr_equal((be.ids, be.offsets, be.word_ids, be.row_ptr), exp, None, f"{name} {data.size} bytes")
    if name == "gpt2_style":
        be = tok.encode_batch_csr(data, off, offsets=False, word_ids=False)
        assert be.offsets is None and be.word_ids is None
        assert np.array_equal(be.ids, exp[0]) and np.array_equal(be.row_ptr, exp[3])
        exp_b = helpers.tiled_expectation(lambda d, o_: o.encode_batch_csr(d, o_, orc.OFF_BYTE), *base, shims)
        be = tok.encode_batch_csr(data, off, byte_offsets=True)
        helpers.assert_csr_equal((be.ids, be.offsets, be.word_ids, be.row_ptr), exp_b, None, f"{name} byte offsets")


@pytest.mark.parametrize("asset", ["gpt2_style", "llama3_style", "wordpiece"])
def test_device_added_tokens_multi_page_warps(asset):
    """added-token extraction on the device (FLAG_ADDED_IDS through the C ABI: a refusal fails the test instead of
    moving the split to the host); ids carry bit 31 on the added tokens, compared in full"""
    tj = helpers.pipeline_json("added_" + asset)
    tok, ref = Tokenizer.from_str(tj), helpers.oracle_backed_tokenizer(tj)
    assert tok._dev_added
    base = helpers.scale_base("added_" + asset, seed=5)
    data, off, shims = helpers.tiled_batch(*base, HOST_BYTES, seed=6)
    assert data.size < 64 << 20
    assert_kb(data.size, asset == "llama3_style", 4)
    exp = helpers.tiled_expectation(lambda d, o_: helpers.host_added_csr(ref, d, o_), *base, shims)
    n_added = int(np.count_nonzero(exp[0] >> 31))
    assert n_added > len(shims) and n_added * 16 <= data.size, "within the device's limit of one span per 16 bytes"
    got = tok._engine_rows(data, off, ALL | _lib.FLAG_ADDED_IDS)
    helpers.assert_csr_equal(got, exp, None, f"device added tokens {asset}")


@pytest.mark.parametrize("name", ["gpt2_style", "wordpiece"])
def test_device_entry_point_larger_warp_ranges(name):
    tj = helpers.pipeline_json(name)
    tok, o = Tokenizer.from_str(tj), oracle(tj)
    base = helpers.scale_base(name, seed=7)
    data, off, shims = helpers.tiled_batch(*base, DEVICE_BYTES, seed=8)
    assert_kb(data.size, False, 6)
    got = helpers.device_csr(tok, data, off, ALL)
    helpers.assert_csr_equal(got, helpers.tiled_expectation(o.encode_batch_csr, *base, shims), None, f"{name} device entry point {data.size} bytes")
