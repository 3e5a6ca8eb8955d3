"""CPU: the pre-tokenization scan (tokenizers_b200/csrc/pretok_logic.cuh) executed on the host by
tests/native/pretok_emul.cpp, composed as the kernels compose it: the bit-plane transposition against its definition,
every claim of the boolean non-ASCII classifier against the class tables (all code points), and the whole scan of all
pre-tokenizers fuzzed against the oracle's regex restatement."""
import ctypes, glob, json, os, subprocess
import numpy as np
import pytest
import helpers, fuzzgen, corpus
from oracle import oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "pretok_emul.cpp")
SO = os.path.join(HERE, "native", "libpretok_emul.so")
HDRS = glob.glob(os.path.join(helpers.ROOT, "tokenizers_b200", "csrc", "*.cuh"))


def _emul():
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(p) for p in [SRC] + HDRS):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC])
    L = ctypes.CDLL(SO)
    L.b2t_emul_pretok.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint32,
                                  ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    L.b2t_emul_check_claims.restype = ctypes.c_uint64
    L.b2t_emul_check_claims.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    L.b2t_emul_check_bitslice.argtypes = [ctypes.c_uint64, ctypes.c_int]
    return L


def _pack2(t):
    t = t.astype(np.uint32).reshape(-1, 16)
    return np.bitwise_or.reduce(t << (np.arange(16, dtype=np.uint32) * 2), axis=1).astype(np.uint32)


def _expected(o, kind, docs, off, n):
    exp = np.zeros(n + 1, dtype=np.uint8); expd = np.zeros(n + 1, dtype=np.uint8)
    for i, d in enumerate(docs):
        base, end = int(off[i]), int(off[i + 1])
        sp = o.pre_tokenize(d)
        if kind in (2, 4):   # Whitespace / BertPreTokenizer: the gaps between the splits are removed whitespace
            pos = 0
            for a, b in sp:
                if a > pos:
                    exp[base + pos] = 1; expd[base + pos] = 1
                exp[base + a] = 1; pos = b
            if pos < end - base:
                exp[base + pos] = 1; expd[base + pos] = 1
        else:
            for a, b in sp:
                exp[base + a] = 1
    return exp[:n], expd[:n]


def test_bitslice_is_a_transposition():
    assert _emul().b2t_emul_check_bitslice(12345, 20000) == 0


@pytest.mark.parametrize("scheme,kind", [("onig", 0), ("onig", 1), ("rust", 2)])
def test_boolean_classifier_never_contradicts_the_table(scheme, kind):
    L = _emul()
    t = np.ascontiguousarray(orc.class_table(scheme), dtype=np.uint8)
    bad = ctypes.c_uint32(0); certain = ctypes.c_uint64(0)
    n_bad = L.b2t_emul_check_claims(kind, t.ctypes.data, ctypes.byref(bad), ctypes.byref(certain))
    assert n_bad == 0, f"{scheme}: {n_bad} wrong claims, first U+{bad.value:04X}"
    # the fast classifier must actually cover the big blocks (Latin, Greek, Cyrillic, CJK, Hangul, emoji)
    assert certain.value > 60000, certain.value


def _straddle_docs(seed, count):
    """Documents dense in multi-byte whitespace, apostrophes and short runs, so that characters and contractions straddle
    32-byte chunk ends in every alignment."""
    rng = np.random.default_rng(seed)
    pieces = [" ", "\u3000", "\u00a0", "\u2003", "\u2028", "  ", "\n", "a", "b's", "'ll", "'re", "'t", "'", "x'", "1",
              "\u00e9", "\u044f", "\u4e2d", "\U0001F600", "\u00d7", "!", "don't", "we've", "I'M", "'S", "\t", "ab",
              "\u0085", "\u1680", "\u0663", "\u2167", "\u00aa", "\u03a9", "\u03f6", "\u4dc5", "\ud55c", "\u2014", "\u3042",
              "\U0001F100", "\u017f", "'\u017f"]
    docs = []
    for _ in range(count):
        k = int(rng.integers(1, 40))
        docs.append("".join(pieces[int(i)] for i in rng.integers(0, len(pieces), k)))
    return docs


def _long_run_docs(seed, count):
    """Documents with digit, newline and whitespace runs of up to 180 bytes between short glue pieces: the runs reach
    past the 64-byte window of the Llama-3 algebra, so its slow path (llama_carry over neighbouring chunks) runs."""
    rng = np.random.default_rng(seed)
    runs = ["1", "\u0663", "\n", "\r\n", " ", "\t", "\u3000", " \n", "\n ", "12 "]
    glue = ["", "a", "ab ", "!", "!!", " x", "'s", "é", "\n", "x1", "中", " "]
    docs = []
    for _ in range(count):
        parts = []
        for _ in range(int(rng.integers(1, 6))):
            parts.append(glue[int(rng.integers(len(glue)))])
            parts.append(runs[int(rng.integers(len(runs)))] * int(rng.integers(1, 60)))
        parts.append(glue[int(rng.integers(len(glue)))])
        docs.append("".join(parts))
    return docs


def _bert_json():
    js = json.loads(helpers.asset_json("wordpiece"))
    js["pre_tokenizer"] = {"type": "BertPreTokenizer"}
    return json.dumps(js)


KINDS = {"gpt2_style": 0, "llama3_style": 1, "wordpiece": 2, "bert_pretok": 4}


def _batches(family):
    if family == "rand":
        return [fuzzgen.rand_docs(seed + s, 600, max_len=60 if s % 3 else 400) for seed in (200, 700) for s in range(6)]
    if family == "corpus":
        return [corpus.to_strings(*corpus.generate(k, seed + k, 0, count)) for seed, count in ((30, 120), (50, 150))
                for k in (1, 2, 4, 5)]
    if family == "straddle":
        return [_straddle_docs(40 + s, 500) for s in range(4)]
    return [_long_run_docs(60 + s, 300) for s in range(4)]


@pytest.mark.parametrize("family", ["rand", "corpus", "straddle", "long_runs"])
@pytest.mark.parametrize("name", list(KINDS))
def test_scan_matches_oracle(name, family):
    L = _emul()
    kind = KINDS[name]
    o = orc.Oracle(_bert_json() if kind == 4 else helpers.asset_json(name))
    tbl = _pack2(orc.class_table({2: "rust", 4: "bert"}.get(kind, "onig")))
    total_gave_back = total_slow = 0
    for docs in _batches(family):
        data, off = helpers.pack_docs(docs)
        n = int(off[-1])
        buf = np.concatenate([data, np.zeros(64, dtype=np.uint8)])
        st = np.zeros(n // 32 + 2, dtype=np.uint32); dr = np.zeros(n // 32 + 2, dtype=np.uint32)
        gave_back = ctypes.c_uint64(0); slow = ctypes.c_uint64(0)
        assert L.b2t_emul_pretok(kind, buf.ctypes.data, n, off.ctypes.data, len(docs), tbl.ctypes.data, st.ctypes.data,
                                 dr.ctypes.data, ctypes.byref(gave_back), ctypes.byref(slow)) == 0
        total_gave_back += gave_back.value; total_slow += slow.value
        bits = np.unpackbits(st.view(np.uint8), bitorder="little")[:n]
        dbits = np.unpackbits(dr.view(np.uint8), bitorder="little")[:n]
        exp, expd = _expected(o, kind, docs, off, n)
        bad = np.nonzero((bits != exp) | (dbits != expd))[0]
        if len(bad):
            di = int(np.searchsorted(off, bad[0], side="right") - 1)
            raise AssertionError(f"{name}: boundary mismatch at byte {bad[0] - int(off[di])} of doc {docs[di]!r}")
    if kind == 0 and family == "straddle":
        assert total_gave_back > 0   # the straddling multi-byte space case was exercised
    if kind == 1 and family == "long_runs":
        assert total_slow > 0        # the Llama-3 slow path was exercised
