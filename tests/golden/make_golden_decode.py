"""Writes golden_decode.json.gz: id rows and the reference wheel's decode_batch of them, for every decoder configuration of
tests/decode_cases.py on a model asset and both skip_special_tokens values, so that the GPU decode tests do not need the
wheel.  Run from the repository root: python tests/golden/make_golden_decode.py"""
import gzip, json, os, sys
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import tokenizers                       # noqa: E402
import decode_cases as dc               # noqa: E402

NAMES = ["gpt2_bytelevel", "llama3_bytelevel", "wordpiece_cleanup", "wordpiece_no_cleanup", "wordpiece_empty_prefix", "wordpiece_no_decoder"]


def main():
    out = {}
    for k, name in enumerate(NAMES):
        tj = dc.tokenizer_json(name)
        ref = tokenizers.Tokenizer.from_str(tj)
        v = ref.get_vocab(with_added_tokens=True)
        n = max(v.values()) + 1
        added = [v[c] for c, _ in dc.ADDED]
        rows = dc.random_rows(100 + k, n, 150, 50, extra=added)
        rows += [[], [v["[SPEC]"]] * 70 + [v["a"], v["the"]], [v["<|sp|>"], v["do not"], v["' x"], v["a"]], [n, 0xFFFFFFFF, (1 << 20) - 1, v["a"]]]
        out[name] = {"rows": rows, "skip": ref.decode_batch(rows, skip_special_tokens=True), "keep": ref.decode_batch(rows, skip_special_tokens=False)}
    with open(os.path.join(HERE, "golden_decode.json.gz"), "wb") as raw, gzip.GzipFile(fileobj=raw, mode="wb", mtime=0) as f:
        f.write(json.dumps({"wheel": tokenizers.__version__, "configs": out}, ensure_ascii=False).encode("utf-8"))


if __name__ == "__main__":
    main()
