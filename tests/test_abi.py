"""CPU: the C-ABI library loads, exports every symbol include/b2t.h declares, and fails loudly without a GPU."""
import ctypes, os, re
import numpy as np
import pytest
import helpers
from tokenizers_b200 import _lib, Tokenizer, UnsupportedConfig, B2TError, parse_tokenizer_json
import json


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(helpers.ROOT, "include", "b2t.h")).read()
    declared = set(re.findall(r"\b(b2t_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    L = _lib.lib()
    for s in declared:
        assert hasattr(L, s), s
    assert b"sm_90a" in L.b2t_version()


def test_unicode_class_tables_match_oracle_tables():
    from oracle import oracle as orc
    L = _lib.lib()
    for scheme, nm in ((0, "onig"), (1, "rust")):
        out = np.zeros(0x110000, dtype=np.uint8)
        assert L.b2t_unicode_class_table(scheme, out.ctypes.data) == 0
        assert np.array_equal(out, orc.class_table(nm))
    assert int((out == 1).sum()) == 144667  # \w (SURVEY.md §7 step 2)


def test_config_detection():
    js = json.loads(helpers.asset_json("gpt2_style"))
    assert parse_tokenizer_json(js)["pretok"] == _lib.PRETOK_BYTELEVEL
    assert parse_tokenizer_json(json.loads(helpers.asset_json("llama3_style")))["pretok"] == _lib.PRETOK_LLAMA3
    assert parse_tokenizer_json(json.loads(helpers.asset_json("wordpiece")))["model"] == _lib.MODEL_WORDPIECE
    bad = dict(js); bad["normalizer"] = {"type": "NFC"}
    with pytest.raises(UnsupportedConfig):
        parse_tokenizer_json(bad)
    bad = json.loads(helpers.asset_json("gpt2_style")); bad["model"]["dropout"] = 0.1
    with pytest.raises(UnsupportedConfig):
        parse_tokenizer_json(bad)
    bad = json.loads(helpers.asset_json("gpt2_style")); bad["pre_tokenizer"] = {"type": "Metaspace"}
    with pytest.raises(UnsupportedConfig):
        parse_tokenizer_json(bad)


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_engine_fails_loudly_without_gpu():
    with pytest.raises(B2TError) as ei:
        Tokenizer.from_str(helpers.asset_json("wordpiece"))
    assert ei.value.code == _lib.B2T_ERR_CUDA and "no CPU path" in str(ei.value)


def test_vocab_errors_are_reported_before_touching_the_gpu():
    j = json.loads(helpers.asset_json("gpt2_style"))
    j["model"]["merges"] = [["zzzz_not_in_vocab", "b"]] + j["model"]["merges"][:10]
    with pytest.raises(B2TError) as ei:
        Tokenizer.from_str(json.dumps(j))
    assert ei.value.code == _lib.B2T_ERR_VOCAB
    j = json.loads(helpers.asset_json("wordpiece")); j["model"]["unk_token"] = "[NOPE]"
    with pytest.raises(B2TError) as ei:
        Tokenizer.from_str(json.dumps(j))
    assert ei.value.code == _lib.B2T_ERR_VOCAB
