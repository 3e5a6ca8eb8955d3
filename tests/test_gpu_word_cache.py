"""GPU (-m gpu): the word cache of the model pass (2^21 slots shared by all blocks of a batch, 4 probes, keys of at most
24 bytes zero-padded with the length in the fingerprint, at most 6 tokens per entry).  A hit must be exact and a miss
harmless: the engine without the cache (B2T_WCACHE=0) matches the oracle, a batch with more distinct words than slots
matches it, and words whose keys differ only where a careless comparison would not look are told apart."""
import random
import numpy as np
import pytest
import helpers, fuzzgen, corpus

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402

# the model pass runs one block per 2 KB page, at most MODEL_MINBLOCKS = 8 of them per SM (csrc/model_kernels.cuh); a
# block looks its pre-tokens up before it publishes them, so only blocks of a later wave can hit what earlier ones published
MODEL_BLOCKS_PER_SM = 8


def engine(tj, wcache=True):
    return helpers.tokenizer_with_env(tj, B2T_WCACHE="1" if wcache else "0")


def csr(tok, data, off):
    be = tok.encode_batch_csr(data, off)
    return be.ids, be.offsets, be.word_ids, be.row_ptr


@pytest.mark.parametrize("name", ["gpt2_style", "llama3_style", "wordpiece"])
def test_cache_off_matches_oracle(name):
    tj = helpers.pipeline_json(name)
    tok, o = engine(tj, wcache=False), orc.Oracle(tj)
    for seed in range(4):
        docs = fuzzgen.rand_docs(5000 + seed, 1500, max_len=60 if seed % 2 else 300)
        helpers.assert_csr_equal(csr(tok, *helpers.pack_docs(docs)), o.encode_batch(docs), docs, f"{name} cache off fuzz {seed}")
    for kind in (1, 2, 4, 5):
        data, off = corpus.generate(kind, 10 + kind, 0, 4000 if kind != 5 else 6000)
        helpers.assert_csr_equal(csr(tok, data, off), o.encode_batch_csr(data, off), corpus.to_strings(data, off), f"{name} cache off corpus {kind}")


def test_cache_off_equals_cache_on_large():
    """48+ MiB tiled GPT-2 batch: with and without the cache, the same output"""
    tj = helpers.pipeline_json("gpt2_style")
    data, off, _ = helpers.tiled_batch(*helpers.scale_base("gpt2_style", seed=9), 50 << 20, seed=10)
    on, off_ = csr(engine(tj), data, off), csr(engine(tj, wcache=False), data, off)
    helpers.assert_csr_equal(off_, on, None, "cache off vs cache on")


def distinct_words(n, seed):
    """n distinct lower-case words of 1..24 letters (most 5..14), as a uint8 matrix [n, 24] and their lengths"""
    rng = np.random.default_rng(seed)
    lens = np.clip(rng.geometric(0.12, size=n + n // 4), 1, 24)
    lens = np.where(lens < 5, rng.integers(5, 15, size=lens.size), lens)
    w = rng.integers(ord("a"), ord("z") + 1, size=(lens.size, 24), dtype=np.uint8)
    w[np.arange(24)[None, :] >= lens[:, None]] = 0
    _, first = np.unique(w.view(np.dtype((np.void, 24))).reshape(-1), return_index=True)
    first = np.sort(first)[:n]
    assert first.size == n
    return w[first], lens[first]


def words_batch(w, lens, per_doc=700):
    """words separated by single spaces, `per_doc` words per document"""
    tok_len = lens + 1
    data = np.full(int(tok_len.sum()), ord(" "), dtype=np.uint8)
    starts = np.concatenate([[0], np.cumsum(tok_len)[:-1]])
    mask = np.arange(24)[None, :] < lens[:, None]
    data[(starts[:, None] + np.arange(24)[None, :])[mask]] = w[mask]
    off = np.concatenate([starts[::per_doc], [data.size]]).astype(np.uint64)
    return data, off


@pytest.mark.parametrize("name", ["gpt2_style", "wordpiece"])
def test_saturated_cache(name):
    """3.3 M distinct pre-tokens: more than the 2^21 slots, every probe sequence fills and later words find no free slot"""
    w, lens = distinct_words(3_300_000, seed=11)
    data, off = words_batch(w, lens)
    assert w.shape[0] > (1 << 21) * 3 // 2 and data.size < 64 << 20
    tj = helpers.pipeline_json(name)
    helpers.assert_csr_equal(csr(engine(tj), data, off), orc.Oracle(tj).encode_batch_csr(data, off), None, f"{name} saturated cache")


def adversary_words(o, sep):
    """words (behind `sep`) whose cache keys differ only in the trailing zero padding, in bytes 21..24, or in the length;
    words that merge into exactly 6 (cached) and 7 (not cached) tokens; long digit runs (never published)"""
    rng = random.Random(12)
    letters = "abcdefghijklmnopqrstuvwxyz"
    out = ["ab", "ab\0", "ab\0\0", "ab\0\0\0\0\0", "\0ab", "a\0b", "x", "x\0", "\0", "\0\0"]
    # keys of 24 bytes that differ in bytes 21..24 only, built from vocabulary words so that they merge into at most 6
    # tokens (a word of more tokens is never cached)
    v5 = sorted(t for t in o.cfg["vocab"] if len(t) == 5 and t.isascii() and t.isalpha() and t.islower())
    v4 = sorted(t for t in o.cfg["vocab"] if len(t) == 4 and t.isascii() and t.isalpha() and t.islower())
    cand = []
    for _ in range(40):
        stem = ("".join(rng.choice(v5) for _ in range(4)))[:20 - len(sep)]
        cand += [stem + rng.choice(v4) for _ in range(6)]
    ids, _, _, rp = o.encode_batch([sep + c for c in cand])
    short = [c for c, t in zip(cand, np.diff(rp.astype(np.int64))) if t <= 6]
    assert len(short) >= 60
    out += short
    for stem in {c[:20 - len(sep)] for c in short[:8]}:
        out += [stem + "wxyz", stem + "wxyz" + "q", stem + "wxy", stem + "wxy\0", stem + "wxyz\0"]   # 23 / 24 / 25 bytes
    cand = ["".join(rng.choice(letters + "é中") for _ in range(rng.randint(8, 16))) for _ in range(4000)]
    ids, _, _, rp = o.encode_batch(cand)
    n_tok = np.diff(rp.astype(np.int64))
    for k in (5, 6, 7):
        picked = [c for c, t in zip(cand, n_tok) if t == k and len(c.encode("utf-8")) <= 24][:12]
        assert len(picked) >= 4, k
        out += picked
    out += ["12345", "123456", "1234567890", "00000", "99999999999999999999"]
    return out


@pytest.mark.parametrize("name", ["gpt2_noregex", "gpt2_style"])
def test_key_adversaries(name):
    """each word thousands of times, in random order, over 8 waves of resident model blocks: the first wave publishes
    every word, the later ones look them up and hit.  Without the regex a document is one pre-token."""
    import torch
    tj = helpers.pipeline_json(name)
    o = orc.Oracle(tj)
    sep = "" if name == "gpt2_noregex" else " "
    words = adversary_words(orc.Oracle(helpers.pipeline_json("gpt2_noregex")), sep)
    wave_bytes = torch.cuda.get_device_properties(0).multi_processor_count * MODEL_BLOCKS_PER_SM * 2048
    mean = np.mean([len((sep + w).encode("utf-8")) for w in words])
    rng = np.random.default_rng(13)
    docs = [sep + words[i] for i in rng.integers(0, len(words), size=int(8 * wave_bytes / mean) + 1)]
    data, off = helpers.pack_docs(docs)
    assert data.size >= 7 * wave_bytes and len(docs) >= 1000 * len(words)
    for wcache in (True, False):
        helpers.assert_csr_equal(csr(engine(tj, wcache), data, off), o.encode_batch_csr(data, off), docs, f"{name} adversaries wcache={wcache}")
