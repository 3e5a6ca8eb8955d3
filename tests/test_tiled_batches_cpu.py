"""The shortcut of the large GPU comparisons (helpers.tiled_batch / tiled_expectation): the output for a batch made of
copies of a base set with shims in between equals the reference's output over the whole batch.  CPU only."""
import numpy as np
import pytest
import helpers
from oracle import oracle as orc

PIPELINES = ["gpt2_style", "gpt2_noregex", "gpt2_prefix", "llama3_style", "wordpiece", "bert_uncased",
             "added_gpt2_style", "added_llama3_style", "added_wordpiece"]


@pytest.mark.parametrize("name", PIPELINES)
def test_tiled_expectation_equals_whole_batch(name):
    tj = helpers.pipeline_json(name)
    slow = name == "bert_uncased" or name.startswith("added_")   # Python normalizer / host added-token logic
    base = helpers.scale_base(name, seed=1, n_corpus=40 if slow else 80, n_fuzz=40 if slow else 80)
    data, off, shims = helpers.tiled_batch(*base, (1 << 20) if slow else (3 << 20), seed=2)
    assert len(set(shims)) > 10 and len(shims) == (len(off) - 1) // (len(base[1]))
    if name.startswith("added_"):
        ref = helpers.oracle_backed_tokenizer(tj)
        encoders = [lambda d, o: helpers.host_added_csr(ref, d, o)]
    else:
        o = orc.Oracle(tj)
        encoders = [lambda d, o_: o.encode_batch_csr(d, o_)]
        if name != "bert_uncased":
            encoders.append(lambda d, o_: o.encode_batch_csr(d, o_, orc.OFF_BYTE))
    for enc in encoders:
        exp = helpers.tiled_expectation(enc, *base, shims)
        whole = enc(data, off)
        helpers.assert_csr_equal(exp, whole, None, f"{name}: tiled expectation vs the whole batch")
        if name.startswith("added_"):
            assert np.count_nonzero(exp[0] >> 31) >= len(shims), "the base set holds added tokens"


def test_kb_formula():
    # 132 SMs: one page pair per warp up to 33 MiB (lean) / 16.5 MiB (Llama-3), then 4
    assert helpers.k1_kb((33 << 20) - 1024, 132, False) == 2 and helpers.k1_kb((33 << 20) + 1024, 132, False) == 4
    assert helpers.k1_kb((33 << 19) - 1024, 132, True) == 2 and helpers.k1_kb((33 << 19) + 1024, 132, True) == 4
    assert helpers.k1_kb(64 << 20, 132, False) == 4 and helpers.k1_kb(1 << 40, 132, False) == 128
