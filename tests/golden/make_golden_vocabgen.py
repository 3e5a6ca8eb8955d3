#!/usr/bin/env python
"""Generate tests/golden/golden_vocabgen.json.gz by running the REFERENCE implementation (the `tokenizers` wheel) on the
generated vocabularies of tests/vocabgen.py: for each configuration the SHA-256 of its tokenizer.json (so a change of the
generators fails loudly instead of comparing against another vocabulary) and the wheel's outputs on a subset of its
documents.

{"<config>": {"sha256": <hex>, "cases": [{"input", "ids", "offsets", "word_ids"}...]}} with char offsets,
add_special_tokens=False.  Deterministic under any PYTHONHASHSEED.
"""
import gzip, hashlib, json, os, sys
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
import vocabgen
from tokenizers import Tokenizer

N_FUZZ = 40


def docs_for(cfg):
    """the documents pinned for `cfg`: its targeted documents of at most 600 bytes and the first N_FUZZ fuzz documents"""
    return [d for d in vocabgen.probes(cfg) if len(d.encode()) <= 600] + vocabgen.fuzz_docs(cfg, N_FUZZ)


def sha256(tj):
    return hashlib.sha256(tj.encode("utf-8")).hexdigest()


if __name__ == "__main__":
    out = {}
    for cfg in vocabgen.CONFIGS:
        tj = cfg.json()
        docs = docs_for(cfg)
        encs = Tokenizer.from_str(tj).encode_batch(docs, add_special_tokens=False)
        out[cfg.name] = {"sha256": sha256(tj),
                         "cases": [{"input": d, "ids": e.ids, "offsets": [list(o) for o in e.offsets], "word_ids": e.word_ids}
                                   for d, e in zip(docs, encs)]}
    path = os.path.join(HERE, "golden_vocabgen.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(json.dumps(out, ensure_ascii=False).encode("utf-8"))
    print("vocabgen", len(out), "configurations", os.path.getsize(path), "bytes")
