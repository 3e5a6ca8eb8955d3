"""Shared test helpers (golden loading, CSR flattening, wheel access)."""
import gzip, json, os
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ASSETS = os.path.join(ROOT, "assets")

GOLDEN_NAMES = ["gpt2", "gpt2_prefix", "llama3", "wordpiece", "bytes_only", "nonmonotone", "ignore_merges"]


def asset_json(name):
    return gzip.open(os.path.join(ASSETS, name + ".json.gz")).read().decode("utf-8")


def _set_path(d, dotted, value):
    ks = dotted.split(".")
    for k in ks[:-1]:
        d = d[k]
    d[ks[-1]] = value


def load_golden(name):
    """-> (tokenizer_json_str, cases)"""
    g = json.loads(gzip.open(os.path.join(GOLDEN, f"golden_{name}.json.gz")).read().decode("utf-8"))
    t = g["tokenizer"]
    if isinstance(t, str) and t.startswith("asset:"):
        tj = asset_json(t[6:])
    elif isinstance(t, dict) and "asset" in t:
        j = json.loads(asset_json(t["asset"]))
        for k, v in t["patch"].items():
            _set_path(j, k, v)
        tj = json.dumps(j)
    else:
        tj = json.dumps(t)
    return tj, g["cases"]


def cases_to_csr(cases):
    ids = np.array([i for c in cases for i in c["ids"]], dtype=np.uint32)
    offs = np.array([o for c in cases for o in c["offsets"]], dtype=np.uint32).reshape(-1, 2)
    wid = np.array([w for c in cases for w in c["word_ids"]], dtype=np.uint32)
    rp = np.zeros(len(cases) + 1, dtype=np.uint64)
    if cases:
        np.cumsum([len(c["ids"]) for c in cases], out=rp[1:])
    return ids, offs, wid, rp


def pack_docs(docs):
    bs = [d.encode("utf-8") for d in docs]
    off = np.zeros(len(bs) + 1, dtype=np.uint64)
    if bs:
        np.cumsum([len(b) for b in bs], out=off[1:])
    return np.frombuffer(b"".join(bs), dtype=np.uint8).copy(), off


def assert_csr_equal(got, exp, docs=None, what=""):
    names = ["ids", "offsets", "word_ids", "row_ptr"]
    for g, e, nm in zip(got, exp, names):
        if g is None:
            continue
        if not np.array_equal(np.asarray(g).reshape(-1), np.asarray(e).reshape(-1)):
            msg = f"{what}: {nm} differ"
            if docs is not None:
                grp, erp = np.asarray(got[3]), np.asarray(exp[3])
                for d in range(len(docs)):
                    a, b = int(erp[d]), int(erp[d + 1])
                    ga, gb = (int(grp[d]), int(grp[d + 1])) if d + 1 < len(grp) else (0, 0)
                    same = (gb - ga == b - a) and all(
                        x is None or np.array_equal(np.asarray(x)[ga:gb], np.asarray(y)[a:b]) for x, y in zip(got[:3], exp[:3]))
                    if not same:
                        msg += f"\n first differing doc {d}: {docs[d]!r}\n  exp ids {np.asarray(exp[0])[a:b].tolist()} off {np.asarray(exp[1])[a:b].tolist()}" \
                               f"\n  got ids {np.asarray(got[0])[ga:gb].tolist()} off {None if got[1] is None else np.asarray(got[1])[ga:gb].tolist()}"
                        break
            raise AssertionError(msg)


def wheel():
    """The reference implementation, if importable here (it is in the dev container and on the GPU image)."""
    try:
        import tokenizers
        return tokenizers
    except Exception:
        return None


def wheel_csr(tok, docs):
    encs = tok.encode_batch(docs, add_special_tokens=False)
    return cases_to_csr([{"ids": e.ids, "offsets": e.offsets, "word_ids": e.word_ids} for e in encs])


# corpus.generate arguments of the large comparison with the reference wheel (golden/wheel_large_digests.json)
WHEEL_LARGE_CORPUS = {"gpt2_style": (2, 99, 0, 40000), "llama3_style": (2, 99, 0, 40000), "wordpiece": (4, 99, 0, 40000)}


def csr_digests(csr):
    """SHA-256 of each CSR array (ids u32, offsets u32 [T, 2], word ids u32, row_ptr u64) and the token count"""
    import hashlib
    dts = (np.uint32, np.uint32, np.uint32, np.uint64)
    d = {nm: hashlib.sha256(np.ascontiguousarray(np.asarray(a).reshape(-1), dtype=dt).tobytes()).hexdigest()
         for nm, a, dt in zip(("ids", "offsets", "word_ids", "row_ptr"), csr, dts)}
    d["n_tokens"] = int(np.asarray(csr[0]).size)
    return d


# ---------------------------------------------------------------------------------------------- host-logic harness
def oracle_backed_tokenizer(tokenizer_json):
    """TEST ONLY: tokenizers_b200.Tokenizer's host logic (added tokens, templates, CSR stitching) in front of the ORACLE
    instead of the GPU engine, so that the host side can be checked on a box without a GPU.  The product class has no
    such switch: it always creates the CUDA engine."""
    import sys
    sys.path.insert(0, ROOT)
    from tokenizers_b200 import _lib
    from tokenizers_b200.tokenizer import Tokenizer
    from oracle.oracle import Oracle, OFF_CHAR, OFF_BYTE

    class OracleBacked(Tokenizer):
        def _create_engine(self, device):
            self._h = None
            self._orc = Oracle(tokenizer_json)

        def _engine_rows(self, data, row_off, flags, zero_copy=False):
            ids, offs, wid, rp = self._orc.encode_batch_csr(data, row_off, OFF_BYTE if flags & _lib.OFFSETS_BYTES else OFF_CHAR)
            return ids, (offs if flags & _lib.WANT_OFFSETS else None), (wid if flags & _lib.WANT_WORD_IDS else None), rp

    return OracleBacked(tokenizer_json)


ADDED_TOKEN_SPECS = [  # (content, single_word, lstrip, rstrip, normalized, special)
    ("<|endoftext|>", False, False, False, False, True),
    ("<mask>", False, True, False, False, True),
    ("[SEP2]", False, False, True, False, True),
    ("<both>", False, True, True, False, True),
    ("tok", True, False, False, True, False),
    ("Zürich", False, False, False, True, False),
    ("<a>", False, False, False, False, True),
    ("<a><b>", False, False, False, False, True),
    ("<|end", False, False, False, True, False),
    ("wörd", True, True, False, False, False),
]


def added_token_entries(vocab, specs):
    """ids the way the reference assigns them (added_vocabulary.rs:281-310): the model's id when the content is already
    in its vocabulary, else the next free id -- what a tokenizer.json written by the reference would contain"""
    nxt, out = len(vocab), []   # get_vocab_size of the model (the assets' vocabularies are dense, so this is also max id + 1)
    for c, sw, ls, rs, nm, sp in specs:
        if c in vocab:
            i = vocab[c]
        else:
            i, nxt = nxt, nxt + 1
        out.append({"id": i, "content": c, "single_word": sw, "lstrip": ls, "rstrip": rs, "normalized": nm, "special": sp})
    return out


def with_added_tokens(tokenizer_json, template=False):
    """asset tokenizer.json + the added tokens above (ids continue after the vocabulary) [+ a TemplateProcessing]"""
    js = json.loads(tokenizer_json)
    n = max(js["model"]["vocab"].values()) + 1
    js["added_tokens"] = added_token_entries(js["model"]["vocab"], ADDED_TOKEN_SPECS)
    if template:
        by = {e["content"]: e["id"] for e in js["added_tokens"]}
        bos, eos = by["<|endoftext|>"], by["<mask>"]
        js["post_processor"] = {"type": "TemplateProcessing",
                                "single": [{"SpecialToken": {"id": "<|endoftext|>", "type_id": 0}}, {"Sequence": {"id": "A", "type_id": 0}},
                                           {"SpecialToken": {"id": "<mask>", "type_id": 0}}],
                                "pair": [{"Sequence": {"id": "A", "type_id": 0}}, {"Sequence": {"id": "B", "type_id": 1}}],
                                "special_tokens": {"<|endoftext|>": {"id": "<|endoftext|>", "ids": [bos], "tokens": ["<|endoftext|>"]},
                                                   "<mask>": {"id": "<mask>", "ids": [eos], "tokens": ["<mask>"]}}}
    return json.dumps(js)


def added_token_docs(seed, n):
    """fuzz documents with the added tokens spliced in: glued to words, surrounded by spaces, back to back, truncated"""
    import random
    from fuzzgen import rand_doc
    rng = random.Random(seed)
    toks = [s[0] for s in ADDED_TOKEN_SPECS]
    docs = ["", "<|endoftext|>", "<|endoftext|><|endoftext|>", "a<|endoftext|>b", "x  <mask>  y", "x [SEP2] \n y", " \t<both>\n ",
            "tok", "a tok b", "atok", "tok.", "toktok", "tok tok", "Zürich", "inZürichx", "<a><b>", "<a><a><b>", "<a", "<|end", "<|endoftext",
            "<|endoftext|", "wörd", " wörd", "xwörd", "wörd!", "  <mask><both>  ", "<mask> tok <both>", "é<mask>é", "toké", "étok", "tok_", "tok1 1tok"]
    while len(docs) < n:
        parts = []
        for _ in range(rng.randint(1, 5)):
            parts.append(rand_doc(rng, 12))
            u = rng.random()
            if u < 0.75:
                t = rng.choice(toks)
                if rng.random() < 0.15:
                    t = t[:rng.randint(1, len(t))]
                parts.append(rng.choice(["", "", " ", "  ", "\n", " "]) + t + rng.choice(["", "", " ", "  ", "\t", "x", "1", "_"]))
        docs.append("".join(parts))
    return docs[:n]
