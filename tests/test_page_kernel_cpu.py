"""The encode path's kernels on the CPU (tests/native/encode_emul.cpp behind the SIMT runtime tests/native/simt.h): the BPE
and WordPiece page kernel in all 40 <MODEL, LAYOUT> instances, the long-pre-token pre-pass (long_find, soft_cut, bpe_long),
the pre-tokenization scan and the scans and compaction around them, run in engine.cu's order, lane by lane with real warp
semantics and several blocks at once, against the oracle.  The runtime's checks (divergent warp syncs, lanes named by a
mask that exited, barriers only some threads reach) are on in every run: a run that trips one fails its test.

Without a GPU the module takes about three minutes on 8 cores (the emulator runs a 2 KB page of the BPE page kernel in
roughly 25 ms; most of the time goes to bpe_long under reordered merges, one merge per round over 1024 fibers).  The last
test compares the engine on the GPU with the emulator, bit for bit, on the same batches."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

import fuzzgen
import helpers
import vocabgen
from helpers import pack_docs, pipeline_json
from oracle import oracle as orc
from tokenizers_b200 import _lib
from tokenizers_b200.tokenizer import engine_config, parse_tokenizer_json

_SO = os.path.join(helpers.ROOT, "tests", "native", "libencode_emul.so")
POISON = 0xDEADBEEF
L_OFFSETS, L_WORD_IDS, L_BYTE_OFFSETS, L_PREFIX, L_ADDED_IDS = 1, 2, 4, 8, 16
ERR_INTERNAL = 4
NORMAL_SLOTS = 1 << 16   # the engine has 2^21; these batches never fill 2^16
SM_COUNT = 2             # soft_cut / bpe_long grids of 8 / 4 blocks: their grid-stride loops take several turns


class _Opts(ctypes.Structure):
    _fields_ = [("layout", ctypes.c_uint32), ("wcache_slots", ctypes.c_uint32), ("wcache_on", ctypes.c_int32), ("sm_count", ctypes.c_int32),
                ("seed", ctypes.c_uint64), ("wc_fp_mask", ctypes.c_uint64)]


_L = None


def lib():
    global _L
    if _L is None:
        L = ctypes.CDLL(_SO)
        L.b2t_emul_create.restype = ctypes.c_void_p
        L.b2t_emul_create.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int]
        L.b2t_emul_destroy.argtypes = [ctypes.c_void_p]
        L.b2t_emul_monotone.argtypes = [ctypes.c_void_p]
        L.b2t_emul_encode.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p]
        L.b2t_emul_error.restype = ctypes.c_char_p
        L.b2t_emul_sizes.argtypes = [ctypes.c_void_p]
        L.b2t_emul_get.argtypes = [ctypes.c_void_p] * 7
        L.b2t_emul_layouts.argtypes = [ctypes.c_void_p]
        _L = L
    return _L


def layouts():
    out = (ctypes.c_uint32 * 64)()
    return list(out[:lib().b2t_emul_layouts(out)])


class Run:
    """one encode of the emulator: the CSR (offsets / word ids hold POISON where the layout writes none), soft_bits, the
    long descriptors of both passes (start, end, pool_off, ntok, soft), the error bits, `stray` (provisional words of an
    output the layout does not write that lost their poison)"""

    def __init__(self, n_docs):
        L = lib()
        sz = (ctypes.c_uint64 * 10)()
        L.b2t_emul_sizes(sz)
        T = sz[0]
        self.ids = np.zeros(T, np.uint32)
        self.offsets = np.zeros((T, 2), np.uint32)
        self.word_ids = np.zeros(T, np.uint32)
        self.row_ptr = np.zeros(n_docs + 1, np.uint64)
        self.soft_bits = np.zeros(sz[3], np.uint32)
        d1, d = np.zeros((sz[1], 4), np.uint64), np.zeros((sz[2], 4), np.uint64)
        L.b2t_emul_get(self.ids.ctypes.data, self.offsets.ctypes.data, self.word_ids.ctypes.data, self.row_ptr.ctypes.data,
                       self.soft_bits.ctypes.data, d1.ctypes.data, d.ctypes.data)
        desc = lambda a: [(int(s), int(e), int(p), int(x & 0xFFFFFFFF), int(x >> 32)) for s, e, p, x in a]
        self.desc1, self.desc = desc(d1), desc(d)
        self.err, self.stray, self.runs = int(sz[4]), int(sz[5]), int(sz[6])

    def csr(self):
        return self.ids, self.offsets, self.word_ids, self.row_ptr

    def soft_positions(self):
        return {w * 32 + b for w in np.flatnonzero(self.soft_bits).tolist() for b in range(32) if (int(self.soft_bits[w]) >> b) & 1}


class Emul:
    """the tables of a tokenizer.json as b2t_engine_create builds them, and the encode pipeline over them"""

    def __init__(self, tj):
        self.tj = tj
        cfg = parse_tokenizer_json(json.loads(tj))
        c, self._keep = engine_config(cfg)
        err = ctypes.create_string_buffer(1024)
        self.h = lib().b2t_emul_create(ctypes.byref(c), err, 1024)
        assert self.h, err.value.decode()
        self.bpe = cfg["model"] == _lib.MODEL_BPE
        self.prefix = bool(cfg["add_prefix_space"])

    def __del__(self):
        if getattr(self, "h", None) and _L is not None:
            _L.b2t_emul_destroy(self.h)

    @property
    def monotone(self):
        return bool(lib().b2t_emul_monotone(self.h))

    def layout(self, byte_offsets=False):
        """the instance the engine picks for offsets + word ids"""
        return L_OFFSETS | L_WORD_IDS | (L_BYTE_OFFSETS if byte_offsets else 0) | (L_PREFIX if self.prefix else 0)

    def encode(self, data, off, layout=None, wcache_slots=NORMAL_SLOTS, wcache_on=1, sm_count=SM_COUNT, seed=1, wc_fp_mask=(1 << 64) - 1):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        off = np.ascontiguousarray(off, dtype=np.uint64)
        o = _Opts(self.layout() if layout is None else layout, wcache_slots, wcache_on, sm_count, seed, wc_fp_mask)
        rc = lib().b2t_emul_encode(self.h, data.ctypes.data, int(off[-1]), off.ctypes.data, len(off) - 1, ctypes.byref(o))
        if rc == 1:
            pytest.fail("SIMT runtime: " + lib().b2t_emul_error().decode())
        assert rc == 0, rc
        r = Run(len(off) - 1)
        assert not (r.err & ERR_INTERNAL), "the page kernel raised ERR_INTERNAL"
        return r


_oracle = {}


def expected(tj, data, off, byte_offsets=False):
    key = (tj, data.tobytes(), off.tobytes(), byte_offsets)
    if key not in _oracle:
        _oracle[key] = orc.Oracle(tj).encode_batch_csr(data, off, orc.OFF_BYTE if byte_offsets else orc.OFF_CHAR)
    return _oracle[key]


def check(em, docs_or_batch, what, **kw):
    """the emulator's CSR (char offsets, and byte offsets) against the oracle"""
    data, off = pack_docs(docs_or_batch) if isinstance(docs_or_batch, list) else docs_or_batch
    docs = docs_or_batch if isinstance(docs_or_batch, list) else None
    for byte in (False, True):
        r = em.encode(data, off, layout=em.layout(byte), **kw)
        helpers.assert_csr_equal(r.csr(), expected(em.tj, data, off, byte), docs, f"{what} byte_offsets={byte}")
    return r


_emuls = {}


def emul(tj):
    if tj not in _emuls:
        _emuls[tj] = Emul(tj)
    return _emuls[tj]


# ------------------------------------------------------------------------------------------------ pipelines
PIPELINES = ["gpt2_style", "gpt2_noregex", "gpt2_prefix", "llama3_style", "wordpiece"]


def corpus_docs(name, seed, n):
    import corpus
    d, o = corpus.generate(4 if name == "wordpiece" else 2, seed, 0, n)
    return corpus.to_strings(d, o)


@pytest.mark.parametrize("name", PIPELINES)
def test_pipelines_match_oracle(name):
    em = emul(pipeline_json(name))
    docs = fuzzgen.rand_docs(61, 250, max_len=200) + corpus_docs(name, 62, 60)
    check(em, docs, name)


CPU_CONFIGS = [c for c in vocabgen.CONFIGS if "bert" not in c.name]   # (BertNormalizer configs: the normalizer is not emulated)


@pytest.mark.parametrize("cfg", CPU_CONFIGS, ids=str)
def test_vocabgen_configs_match_oracle(cfg):
    """the configuration's probes and fuzz documents; BPE: soft_bits of every long pre-token == vocabgen.soft_cuts, and
    LongDesc.soft"""
    em = emul(cfg.json())
    docs = vocabgen.probes(cfg) + vocabgen.fuzz_docs(cfg, 120)
    r = check(em, docs, cfg.name)
    if em.bpe:
        data, off = pack_docs([(" " + d if em.prefix and d and d[0] != " " else d) for d in docs])   # the re-packed batch
        assert r.desc1
        check_soft_bits(em, r, data)
        if cfg.kwargs.get("pretok") == "noregex":
            check_long_desc(r, set(off.tolist()), data)


# ------------------------------------------------------------------------------------------------ layouts
def layout_batch(model):
    rng = random.Random(5)
    probes = helpers.bpe_probes() if model == "bpe" else helpers.wordpiece_probes(100)
    docs = helpers.place([(p, k * helpers.PAGE + rng.choice(helpers.EDGES) + rng.choice([-1, 0, 1]), rng.choice(["start", "end"]))
                          for k, p in enumerate(probes, start=1)], "doc")
    return docs + fuzzgen.rand_docs(71, 120, max_len=120) + [""] * 3


@pytest.mark.parametrize("model", ["bpe", "wordpiece"])
def test_every_layout(model):
    """all 20 instances of the model: what the layout writes equals the oracle, what it does not write keeps its poison"""
    docs = layout_batch(model)
    data, off = pack_docs(docs)
    lays = layouts()
    assert len(lays) == 20 and len(set(lays)) == 20
    for lay in lays:
        name = ("gpt2_prefix" if lay & L_PREFIX else "gpt2_style") if model == "bpe" else "wordpiece"
        em = emul(pipeline_json(name))
        r = em.encode(data, off, layout=lay, seed=lay + 1)
        exp = expected(em.tj, data, off, bool(lay & L_BYTE_OFFSETS))
        what = f"{model} layout {lay}"
        assert r.stray == 0, f"{what}: the page kernel wrote an output the layout does not have"
        assert np.array_equal(r.ids, exp[0]) and np.array_equal(r.row_ptr, exp[3]), what
        if lay & L_OFFSETS:
            assert np.array_equal(r.offsets, exp[1]), what
        else:
            assert (r.offsets == POISON).all(), what
        if lay & L_WORD_IDS:
            assert np.array_equal(r.word_ids, exp[2]), what
        else:
            assert (r.word_ids == POISON).all(), what


# ------------------------------------------------------------------------------------------------ edges
def words_of_tokens(tj, counts, n_each=2, seed=9):
    """letter words of <= 24 bytes (one GPT-2 pre-token each) whose BPE result has exactly `count` tokens"""
    rng = random.Random(seed)
    o = orc.Oracle(tj)
    found = {c: [] for c in counts}
    while any(len(v) < n_each for v in found.values()):
        w = "".join(rng.choice("qxzjkvwyfbpgQXZJ") for _ in range(rng.randint(8, 24)))
        data, off = pack_docs([w])
        k = len(o.encode_batch_csr(data, off)[0])
        if k in found and len(found[k]) < n_each:
            found[k].append(w)
    return [w for c in counts for w in found[c]]


def edge_probes(tj, model):
    rng = random.Random(4)
    out = [helpers.word(rng, n, w) for n in (16, 17, 24, 25, 32, 33) for w in (1, 2, 4)]
    out += [helpers.word(rng, n, w) for n in (256, 257) for w in (1, 3)]
    if model == "bpe":
        out += words_of_tokens(tj, (6, 7))
    return out


@pytest.mark.parametrize("name", ["gpt2_style", "wordpiece"])
def test_pretoken_lengths_at_page_edges(name):
    """pre-tokens of exactly 16/17, 24/25, 32/33 and 256/257 bytes and word-cache results of 6 and 7 tokens, each across
    page edges, at document starts and among empty documents; every probe twice, so the second occurrence can hit"""
    tj = pipeline_json(name)
    em = emul(tj)
    probes = edge_probes(tj, "bpe" if name != "wordpiece" else "wp")
    slots = [(p, k * helpers.PAGE + e + d, a) for k, (p, e, d, a) in enumerate(
        ((p, e, d, a) for p in probes for e, d, a in ((0, 0, "start"), (0, -1, "end"), (32, 1, "start"), (256, 0, "end"))), start=1)]
    docs = helpers.place(slots, "doc")
    docs = [d for x in docs for d in (x, "")] + helpers.place(slots[::3], "text") + [" " + p for p in probes] * 2
    check(em, docs, name)


# ------------------------------------------------------------------------------------------------ word cache
def repeat_batch(seed, n_docs=400):
    """a batch where most pre-tokens repeat: a small lexicon, words of 1..30 bytes, across ~25 pages"""
    rng = random.Random(seed)
    lex = ["".join(rng.choice("abcdefghijklmnopqrstuvwxyzéж") for _ in range(rng.randint(1, 14))) for _ in range(60)]
    lex += ["".join(rng.choice("qxzjkvw") for _ in range(rng.randint(15, 24))) for _ in range(10)]
    return [" ".join(rng.choice(lex) for _ in range(rng.randint(1, 30))) for _ in range(n_docs)]


@pytest.mark.parametrize("name", ["gpt2_style", "llama3_style", "wordpiece"])
def test_word_cache_on_off_and_tiny(name):
    """cache off, the normal cache and a cache of 16 slots (every probe chain fills and collides) give the oracle's result"""
    em = emul(pipeline_json(name))
    data, off = pack_docs(repeat_batch(3))
    exp = expected(em.tj, data, off)
    for kw in (dict(wcache_on=0), dict(), dict(wcache_slots=16), dict(wcache_slots=16, seed=0)):
        r = em.encode(data, off, **kw)
        helpers.assert_csr_equal(r.csr(), exp, None, f"{name} {kw}")


@pytest.mark.parametrize("name", ["gpt2_style", "wordpiece"])
def test_word_cache_hit_needs_the_whole_key(name):
    """pre-tokens of 17..24 bytes with at most 6 tokens (so the cache holds them) that share their first 16 bytes, with
    every fingerprint colliding: a hit then rests on the comparison of all 24 key bytes (with real fingerprints two such
    words never meet in a slot)"""
    tj = pipeline_json(name)
    em = emul(tj)
    rng = random.Random(8)
    o = orc.Oracle(tj)
    ntok = lambda w: len(o.encode_batch_csr(*pack_docs([" " + w]))[0])
    short = [w for w in ["the", "and", "of", "to", "in", "is", "it", "that", "was", "for", "on", "as", "with", "he", "be", "at", "by",
                         "his", "her", "not", "are", "this", "from", "had", "but"] if ntok(w) == 1]
    hl = 15 if name == "gpt2_style" else 16   # (GPT-2: the pre-token is " " + word)
    heads = []
    while len(heads) < 2:
        h = ""
        while len(h) < hl:
            h += rng.choice(short)
        if len(h) == hl and ntok(h) <= 4 and h not in heads:
            heads.append(h)
    words = sorted({h + "".join(rng.choice(short) for _ in range(rng.randint(1, 2))) for h in heads for _ in range(60)})
    words = [w for w in words if len(w) <= hl + 8 and ntok(w) <= 6]
    assert len(words) >= 12
    docs = [" ".join(rng.choice(words) for _ in range(rng.randint(1, 12))) for _ in range(300)]
    data, off = pack_docs(docs)
    for slots in (NORMAL_SLOTS, 16, 4):   # (4 slots: every look-up probes the whole table)
        r = em.encode(data, off, wcache_slots=slots, wc_fp_mask=0)
        helpers.assert_csr_equal(r.csr(), expected(em.tj, data, off), docs, f"{name} colliding fingerprints, {slots} slots")


@pytest.mark.parametrize("seed", [2, 3, 4])
def test_word_cache_handover_between_blocks(seed):
    """several blocks run at once over a batch of repeated words: slots are claimed (BUSY), published (READY) and read by
    other blocks while they are being written, in a different lane order per seed"""
    em = emul(pipeline_json("gpt2_style"))
    data, off = pack_docs(repeat_batch(10 + seed, 600))
    for slots in (NORMAL_SLOTS, 64):
        r = em.encode(data, off, wcache_slots=slots, seed=seed)
        helpers.assert_csr_equal(r.csr(), expected(em.tj, data, off), None, f"seed {seed} slots {slots}")


# ------------------------------------------------------------------------------------------------ soft cuts
def bpe_json(merges, pretok="noregex", ignore_merges=False, extra=()):
    """byte-level BPE over all 256 bytes, the given merges (raw byte strings) in rank order, and vocabulary-only tokens"""
    toks = [bytes([b]) for b in range(256)]
    for a, b in merges:
        if a + b not in toks:
            toks.append(a + b)
    toks += [t for t in extra if t not in toks]
    vocab = {vocabgen.byte_level(t): i for i, t in enumerate(toks)}
    model = {"type": "BPE", "dropout": None, "unk_token": None, "continuing_subword_prefix": None, "end_of_word_suffix": None,
             "fuse_unk": False, "byte_fallback": False, "ignore_merges": ignore_merges, "vocab": vocab,
             "merges": [[vocabgen.byte_level(a), vocabgen.byte_level(b)] for a, b in merges]}
    return json.dumps({"version": "1.0", "truncation": None, "padding": None, "added_tokens": [], "normalizer": None,
                       "pre_tokenizer": vocabgen.PRETOKENIZERS[pretok], "post_processor": None, "decoder": None, "model": model},
                      ensure_ascii=False)


def vocab_bytes(tj):
    return [vocabgen.from_byte_level(t) for t in json.loads(tj)["model"]["vocab"]]


# "pq": held together by the 2-byte token only; "klm": l|m held by the left triple only; "uvw" (u + vw): u|v held by the
# right triple only.  A pre-token that starts "uv" has its u|v boundary at s + 1 (no left triple), one that ends "uv" at
# e - 1 (no right triple: cut).
SOFT_MERGES = [(b"p", b"q"), (b"k", b"l"), (b"kl", b"m"), (b"v", b"w"), (b"u", b"vw"), (b"m", b"m"), (b"mm", b"mm")]


def soft_docs(seed, n):
    rng = random.Random(seed)
    parts = ["pq", "klm", "uvw", "uv", "vw", "kl", "lm", ".", "..", "m", "mmmm", "q", "u", "w"]
    docs = []
    for i in range(n):
        body = "".join(rng.choice(parts) for _ in range(rng.randint(120, 400)))
        docs.append(["uvw", "uv", "..", "pq", ""][i % 5] + body + ["uv", "kl", "uvw", ".", "q"][(i // 5) % 5])
    return docs + ["x" * 10, ""]


def check_soft_bits(em, r, data):
    tokens = vocab_bytes(em.tj)
    got = r.soft_positions()
    want = set()
    raw = data.tobytes()
    for s, e, *_ in r.desc1:
        assert e - s > 256
        a = s
        for piece in vocabgen.soft_cuts(tokens, raw[s:e])[:-1]:
            a += len(piece)
            want.add(a)
    assert got == want, f"soft_bits differ from vocabgen.soft_cuts: missing {sorted(want - got)[:8]}, extra {sorted(got - want)[:8]}"


def check_long_desc(r, starts, data):
    """a piece of a cut pre-token starts or ends at a soft cut: LongDesc.soft"""
    n = len(data)
    for s, e, _pool, _ntok, soft in r.desc:
        real = s in starts and (e in starts or e == n)
        assert soft == (0 if real else 1), (s, e, soft)


def test_soft_cuts_match_restatement():
    pretok = "noregex"   # (the whole document is one pre-token)
    tj = bpe_json(SOFT_MERGES, pretok=pretok)
    em = emul(tj)
    docs = soft_docs(1, 30)
    data, off = pack_docs(docs)
    r = em.encode(data, off)
    helpers.assert_csr_equal(r.csr(), expected(tj, data, off), docs, f"soft cuts {pretok}")
    assert len(r.desc1) >= 20
    check_soft_bits(em, r, data)
    check_long_desc(r, set(off.tolist()), data)


def test_ignore_merges_whole_token_against_cut_pretoken():
    """ignore_merges: a long pre-token that is one vocabulary token is that token (soft = 0, one token); the same bytes
    with a cut in them are merged piece by piece"""
    tok = b"QRSTUV" * 50   # 300 bytes, vocabulary-only
    tj = bpe_json(SOFT_MERGES, ignore_merges=True, extra=[tok])
    em = emul(tj)
    docs = [tok.decode(), tok.decode() + ".", "!" + tok.decode(), (b"QRSTUV" * 25).decode() + "pq" + (b"QRSTUV" * 25).decode()]
    data, off = pack_docs(docs)
    r = em.encode(data, off)
    helpers.assert_csr_equal(r.csr(), expected(tj, data, off), docs, "ignore_merges")
    assert int(r.row_ptr[1]) == 1
    whole = [d for d in r.desc if d[0] == 0]
    assert whole and whole[0][4] == 0 and whole[0][3] == 1


# ------------------------------------------------------------------------------------------------ long merges
SYMBOLS = {"a": [], "é": [(b"\xc3", b"\xa9")], "xyz": [(b"x", b"y"), (b"xy", b"z")]}


def chain_merges(sym_merges, sym, top=512):
    out = list(sym_merges)
    t = sym
    while 2 * len(t) <= top:
        out.append((t, t))
        t += t
    return out


def long_run_merges(shuffle_seed=None):
    """doubling chains of a one-byte symbol, a two-byte one and a three-byte one; "b" + "a" and "a" + "c" rank before
    the chain of "a", so a run of a's behind a "b" or in front of a "c" is broken by an earlier merge"""
    m = [(b"b", b"a"), (b"a", b"c")]
    for s, sm in SYMBOLS.items():
        m += chain_merges(sm, s.encode())
    if shuffle_seed is not None:
        random.Random(shuffle_seed).shuffle(m)
    return m


def run_docs(max_len):
    out = []
    for s in SYMBOLS:
        w = len(s.encode())
        for nb in (257, 258, 300, 301, 511, 512, 513, 1023, 1024, 1025, 2047, 2999, 3000):
            if nb <= max_len:
                k = nb // w
                out += [s * k, s * (k + 1)]   # odd and even run lengths (in symbols)
    for k in (257, 300, 511, 1000, 2999):
        if k + 2 <= max_len:
            out += ["b" + "a" * k, "ba" * 3 + "a" * k, "a" * k + "c", "b" + "a" * k + "c" + "a" * (k // 2), "a" * (k // 3) + "é" * (k // 3)]
    return out


@pytest.mark.parametrize("monotone", [True, False])
def test_long_runs(monotone):
    """x == y runs of 257..3000 bytes of 1-, 2- and 3-byte symbols, odd and even, broken by an earlier merge, under a
    monotone table (every occurrence of the minimal pair per round, parity from the run start) and under the same merges
    reordered (one merge per round; runs up to 1025 bytes to keep the emulator fast)"""
    merges = long_run_merges(None if monotone else 7)
    tj = bpe_json(merges)
    em = emul(tj)
    vocab = json.loads(tj)["model"]["vocab"]
    strs = [(vocabgen.byte_level(a), vocabgen.byte_level(b)) for a, b in merges]
    assert em.monotone == vocabgen.is_monotone(vocab, strs) == monotone
    docs = run_docs(3000 if monotone else 1025)
    data, off = pack_docs(docs)
    r = em.encode(data, off)
    helpers.assert_csr_equal(r.csr(), expected(tj, data, off), docs, f"long runs monotone={monotone}")
    assert len(r.desc) >= len(docs) - 2


def all_bpe_tables():
    out = [(c.name, c.json()) for c in vocabgen.CONFIGS if c.kind == "bpe"]
    out += [(n, pipeline_json(n)) for n in ("gpt2_style", "llama3_style")]
    out += [("soft", bpe_json(SOFT_MERGES)), ("runs", bpe_json(long_run_merges())), ("runs_shuffled", bpe_json(long_run_merges(7)))]
    out += [(f"runs_shuffled_{s}", bpe_json(long_run_merges(s))) for s in range(3)]
    return out


def test_monotone_flag_equals_restatement():
    """host_tables.cu's monotone flag (which decides whether bpe_long merges every occurrence per round) == vocabgen.is_monotone"""
    seen = set()
    for name, tj in all_bpe_tables():
        m = json.loads(tj)["model"]
        merges = [tuple(x.split(" ")) if isinstance(x, str) else tuple(x) for x in m["merges"]]
        want = vocabgen.is_monotone(m["vocab"], merges)
        assert Emul(tj).monotone == want, name
        seen.add(want)
    assert seen == {True, False}


# ------------------------------------------------------------------------------------------------ GPU cross-check
def cross_batches():
    out = [(n, layout_batch("wordpiece" if n == "wordpiece" else "bpe")) for n in PIPELINES]
    out += [("repeat", repeat_batch(3)), ("runs", run_docs(3000)), ("soft", soft_docs(1, 30))]
    return out


@pytest.mark.gpu
def test_engine_equals_emulator_every_layout():
    """the engine on the GPU and encode_emul give the same bits for every layout the engine can form, on the same
    batches: encode_emul keeps following engine.cu"""
    from tokenizers_b200 import Tokenizer
    sm_count = None
    for name, docs in cross_batches():
        tj = {"repeat": pipeline_json("gpt2_style"), "runs": bpe_json(long_run_merges()), "soft": bpe_json(SOFT_MERGES)}.get(name) or pipeline_json(name)
        em = emul(tj)
        tok = Tokenizer.from_str(tj)
        if sm_count is None:
            import torch
            sm_count = torch.cuda.get_device_properties(0).multi_processor_count   # (the engine's grids of K1, soft_cut and bpe_long)
        data, off = pack_docs(docs)
        for lay in layouts():
            if lay & L_ADDED_IDS or bool(lay & L_PREFIX) != (em.prefix and bool(lay & L_OFFSETS)):
                continue   # (no added tokens here; the engine takes the prefix mapping exactly when it has offsets to map)
            be = tok.encode_batch_csr(data, off, offsets=bool(lay & L_OFFSETS), word_ids=bool(lay & L_WORD_IDS), byte_offsets=bool(lay & L_BYTE_OFFSETS))
            r = em.encode(data, off, layout=lay, sm_count=sm_count, wcache_slots=1 << 21)
            what = f"{name} layout {lay}"
            assert np.array_equal(be.ids, r.ids) and np.array_equal(be.row_ptr, r.row_ptr), what
            if lay & L_OFFSETS:
                assert np.array_equal(np.asarray(be.offsets).reshape(-1, 2), r.offsets), what
            if lay & L_WORD_IDS:
                assert np.array_equal(be.word_ids, r.word_ids), what
