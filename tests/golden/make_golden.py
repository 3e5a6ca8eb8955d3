#!/usr/bin/env python
"""Generate tests/golden/golden_*.json.gz by running the REFERENCE implementation (the `tokenizers` wheel, same Rust core
as huggingface/tokenizers) on seeded inputs.  The outputs are committed and are what pins the
oracle (and, through it, the CUDA path) on boxes where the wheel is not consulted.

Each file: {"tokenizer": <tokenizer.json dict or asset name>, "cases": [{"input", "ids", "offsets", "word_ids"}...]}
with char offsets, add_special_tokens=False (== Tokenizer.encode_batch of the Python binding).
"""
import gzip, json, os, sys
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "..", "tools"))
import fuzzgen, corpus
from tokenizers import Tokenizer, models, pre_tokenizers

ASSETS = os.path.join(HERE, "..", "..", "assets")


def byte_alphabet():
    return sorted(pre_tokenizers.ByteLevel.alphabet())


def tiny_bytelevel(merges, extra_tokens, add_prefix_space=False, ignore_merges=False):
    vocab = {c: i for i, c in enumerate(byte_alphabet())}
    for t in extra_tokens:
        vocab[t] = len(vocab)
    tok = Tokenizer(models.BPE(vocab=vocab, merges=merges, ignore_merges=ignore_merges))
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=add_prefix_space)
    return json.loads(tok.to_str())


def cases_for(tok, docs):
    encs = tok.encode_batch(docs, add_special_tokens=False)
    return [{"input": d, "ids": e.ids, "offsets": [list(o) for o in e.offsets], "word_ids": e.word_ids} for d, e in zip(docs, encs)]


def dump(name, tokenizer_field, tok, docs):
    path = os.path.join(HERE, f"golden_{name}.json.gz")
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(json.dumps({"tokenizer": tokenizer_field, "cases": cases_for(tok, docs)}, ensure_ascii=False).encode("utf-8"))
    print(name, len(docs), "cases", os.path.getsize(path), "bytes")


def asset(name):
    return gzip.open(os.path.join(ASSETS, name + ".json.gz")).read().decode("utf-8")


def docs_for(seed, kind):
    d = fuzzgen.rand_docs(seed, 160, max_len=40)
    data, off = corpus.generate(kind, 900 + seed, 0, 12)
    return d + corpus.to_strings(data, off)


MICRO = ["a's", "1's", "\n's", " 's", "!'s", "'s's", "''s", "a  's", "a'S", "a'sb", "a'llve", "a're's", "a'r", "  a", "a  ", "a \n b",
         "a\n\nb", "a \t", "\t a", "a b", "a  b", "12 34", " 1a", "a1 ", "!! ?", "1234567", "a'S b", " \n \n  x", "!!\n\nx",
         "'xab", "a\r\nb", "  \n", "x  \n  y", "\thello", "-hello", "1a2", "i⭢j é", "😀a", "", "hello é world! héllo " + "a" * 101]

if __name__ == "__main__":
    js = asset("gpt2_style"); dump("gpt2", "asset:gpt2_style", Tokenizer.from_str(js), docs_for(1, 2) + MICRO)
    j = json.loads(js); j["pre_tokenizer"]["add_prefix_space"] = True
    dump("gpt2_prefix", {"asset": "gpt2_style", "patch": {"pre_tokenizer.add_prefix_space": True}}, Tokenizer.from_str(json.dumps(j)), docs_for(2, 2)[:80] + MICRO)
    js = asset("llama3_style"); dump("llama3", "asset:llama3_style", Tokenizer.from_str(js), docs_for(3, 2) + MICRO)
    js = asset("wordpiece"); dump("wordpiece", "asset:wordpiece", Tokenizer.from_str(js), docs_for(4, 4) + MICRO)
    # byte-level BPE without merges: tokens are bytes (pins the offset algebra, tests/offsets.rs:45-54)
    t = tiny_bytelevel([], []); dump("bytes_only", t, Tokenizer.from_str(json.dumps(t)), MICRO + fuzzgen.rand_docs(5, 60, 30))
    # hand-written, NON-monotone merges: (ab,a) ranks before (a,b); exercises the heap order of word.rs:162-250
    t = tiny_bytelevel([("ab", "a"), ("a", "b"), ("b", "a"), ("aba", "b"), ("a", "a"), ("aa", "a")], ["ab", "aba", "ba", "abab", "aa", "aaa"])
    dump("nonmonotone", t, Tokenizer.from_str(json.dumps(t)),
         ["abab", "ababab", "aaa", "aaaa", "aaaaa", "baba", "abaab", "aabab abab", "ab", "a", "bab", "aabbaabb", "abababababababab" * 3, "aaaaaaaaaaaaaaaaaaaaaaaaaaaaaaaaaaaaa"])
    # ignore_merges on a tiny vocab (models/bpe/model.rs:1077-1169 test_ignore_merges)
    t = tiny_bytelevel([("a", "b"), ("ab", "c")], ["ab", "abc", "Ġabc", "bc"], ignore_merges=True)
    dump("ignore_merges", t, Tokenizer.from_str(json.dumps(t)), ["abc", " abc", "abc abc", "bc", "abcabc", "ab c", "Ġabc"])
