#!/usr/bin/env python
"""SHA-256 digests of the reference wheel's CSR (ids, char offsets, word ids, row_ptr) for the 40 k-document corpora of
test_gpu_parity.py::test_gpu_matches_reference_wheel_large -- too large to store, so the test compares digests:
python tests/golden/make_golden_wheel_large.py  ->  tests/golden/wheel_large_digests.json"""
import json, os, sys
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, os.path.join(ROOT, "tools"))
import tokenizers                       # noqa: E402
import corpus, helpers                  # noqa: E402


def main():
    out = {"wheel": tokenizers.__version__}
    for name in ("gpt2_style", "llama3_style", "wordpiece"):
        data, off = corpus.generate(*helpers.WHEEL_LARGE_CORPUS[name])
        csr = helpers.wheel_csr(tokenizers.Tokenizer.from_str(helpers.asset_json(name)), corpus.to_strings(data, off))
        out[name] = helpers.csr_digests(csr)
    path = os.path.join(HERE, "wheel_large_digests.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(path, out)


if __name__ == "__main__":
    main()
