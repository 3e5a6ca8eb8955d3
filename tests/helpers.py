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


def tokenizer_with_env(tokenizer_json, **env):
    """tokenizers_b200.Tokenizer created with the engine switches in `env` (B2T_WCACHE, B2T_CHUNK_BYTES: read when the
    engine is created); the caller's environment is restored afterwards"""
    from tokenizers_b200 import Tokenizer
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return Tokenizer.from_str(tokenizer_json)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def device_csr(tok, data, doc_off, flags):
    """b2t_encode_batch_device: the batch already on the GPU, the result left there; copied back to host arrays
    (ids, offsets or None, word ids or None, row_ptr) to compare"""
    import ctypes
    import torch
    from tokenizers_b200 import _lib
    d_bytes = torch.from_numpy(np.ascontiguousarray(data, dtype=np.uint8)).cuda()
    d_off = torch.from_numpy(np.asarray(doc_off).astype(np.int64)).cuda()
    L = _lib.lib()
    res = ctypes.c_void_p()
    _lib.check(L.b2t_encode_batch_device(tok.handle, d_bytes.data_ptr(), int(doc_off[-1]), d_off.data_ptr(), len(doc_off) - 1, flags, None,
                                         ctypes.byref(res)))
    try:
        assert L.b2t_result_on_device(res) == 1
        T = L.b2t_result_n_tokens(res)
        cudart = ctypes.CDLL("libcudart.so")
        torch.cuda.synchronize()

        def dev(ptr, count, dtype):
            out = np.empty(count, dtype=dtype)
            if count:
                assert cudart.cudaMemcpy(ctypes.c_void_p(out.ctypes.data), ctypes.c_void_p(ptr), ctypes.c_size_t(out.nbytes), 2) == 0  # device -> host
            return out
        return (dev(L.b2t_result_ids(res), T, np.uint32),
                dev(L.b2t_result_offsets(res), 2 * T, np.uint32).reshape(-1, 2) if flags & _lib.WANT_OFFSETS else None,
                dev(L.b2t_result_word_ids(res), T, np.uint32) if flags & _lib.WANT_WORD_IDS else None,
                dev(L.b2t_result_row_ptr(res), len(doc_off), np.uint64))
    finally:
        L.b2t_result_free(res)


def host_added_csr(ref, data, doc_off, byte_offsets=False):
    """What the device extraction (FLAG_ADDED_IDS) must return, from `ref` = oracle_backed_tokenizer(...): the host split
    (added.py) in front of the oracle, with bit 31 set on the ids of the added tokens found in the text"""
    from tokenizers_b200 import _lib, added
    flags = _lib.WANT_OFFSETS | _lib.WANT_WORD_IDS | (_lib.OFFSETS_BYTES if byte_offsets else 0)
    row_off, parts, cut = added.split_batch(ref._added, data, doc_off)
    ids, offs, wid, rp = ref._engine_rows(data, row_off, flags)
    if cut:
        ids, offs, wid, rp, added_at = added.stitch_rows(data, doc_off, parts, ids, offs, wid, rp, byte_offsets)
        ids = np.array(ids, dtype=np.uint32)
        ids[[i for i, _, _ in added_at]] |= np.uint32(1 << 31)
    return ids, offs, wid, rp


# ------------------------------------------------------------------------------------------------- tiled batches
# Tokenization is per document, so a batch made of copies of one base set of documents, with a short "shim" document of
# varying length in front of every copy, has an output that is the base set's output repeated (with the shims' in
# between): the reference runs once per base set and once per distinct shim, not over the whole batch.  The shims move
# every copy to a different offset relative to the 32 B chunks, 1 KB iterations, 2 KB pages and warp ranges.
SHIM_TEXT = b"the shim moves the next copy along; "


def shim_doc(r):
    return (SHIM_TEXT * (r // len(SHIM_TEXT) + 1))[:r]


def tiled_batch(base_data, base_off, target_bytes, seed=0, shim_max=2048):
    """-> (data uint8, doc_off uint64, shims): [shim(shims[0]), base..., shim(shims[1]), base..., ...] of at least
    target_bytes; shim lengths are drawn from 0..shim_max-1"""
    rng = np.random.default_rng(seed)
    base_data = np.asarray(base_data, dtype=np.uint8)
    base_off = np.asarray(base_off, dtype=np.uint64)
    nb = int(base_off[-1])
    copies = max(1, -(-int(target_bytes) // (nb + shim_max // 2)))
    shims = rng.integers(0, shim_max, size=copies).tolist()
    data = np.empty(sum(shims) + copies * nb, dtype=np.uint8)
    nd = len(base_off) - 1
    off = np.empty(copies * (nd + 1) + 1, dtype=np.uint64)
    pos, k = 0, 0
    for r in shims:
        data[pos:pos + r] = np.frombuffer(shim_doc(r), dtype=np.uint8)
        off[k] = pos
        pos += r
        off[k + 1:k + 1 + nd] = base_off[:-1] + np.uint64(pos)
        data[pos:pos + nb] = base_data
        pos += nb
        k += nd + 1
    off[k] = pos
    return data, off, shims


def tiled_expectation(encode, base_data, base_off, shims):
    """The output of `encode(data, doc_off) -> (ids, offsets | None, word_ids | None, row_ptr)` for tiled_batch(...),
    from one call on the base set and one per distinct shim length"""
    base = encode(np.asarray(base_data, dtype=np.uint8), np.asarray(base_off, dtype=np.uint64))
    per_shim = {}
    for r in set(shims):
        b = np.frombuffer(shim_doc(r), dtype=np.uint8).copy()
        per_shim[r] = encode(b, np.array([0, r], dtype=np.uint64))
    parts = [[] for _ in range(3)]
    counts = []
    for r in shims:
        for piece in (per_shim[r], base):
            for k in range(3):
                if piece[k] is not None:
                    parts[k].append(np.asarray(piece[k]))
            counts.append(np.diff(np.asarray(piece[3], dtype=np.uint64)))
    out = [np.concatenate(p) if p else None for p in parts]
    rp = np.zeros(sum(len(c) for c in counts) + 1, dtype=np.uint64)
    np.cumsum(np.concatenate(counts), out=rp[1:])
    return out[0], out[1], out[2], rp


def k1_kb(n_bytes, sm_count, llama3):
    """KB of the batch that each warp of the pre-tokenization scan (K1) owns: the formula of launch_pretok in
    tokenizers_b200/csrc/engine.cu (the lean kernel runs 8 blocks of 4 warps per SM, the Llama-3 kernel 4)"""
    n_kb = (n_bytes // 32 + 1 + 31) // 32
    resident = sm_count * (4 if llama3 else 8) * 4
    kb = -(-n_kb // (4 * resident))
    return min(128, max(2, (kb + 1) & ~1))


def bert_json(flags):
    """the wordpiece asset behind BertNormalizer(**flags) + BertPreTokenizer: the bert-base pipeline"""
    js = json.loads(asset_json("wordpiece"))
    js["normalizer"] = dict(type="BertNormalizer", **flags)
    js["pre_tokenizer"] = {"type": "BertPreTokenizer"}
    return json.dumps(js)


BERT_UNCASED = dict(clean_text=True, handle_chinese_chars=True, strip_accents=None, lowercase=True)


def pipeline_json(name):
    """tokenizer.json of the pipelines the scale and edge tests run"""
    if name in ("gpt2_style", "llama3_style", "wordpiece"):
        return asset_json(name)
    if name in ("gpt2_noregex", "gpt2_prefix"):
        j = json.loads(asset_json("gpt2_style"))
        j["pre_tokenizer"].update({"use_regex": False} if name == "gpt2_noregex" else {"add_prefix_space": True})
        return json.dumps(j)
    if name == "bert_uncased":
        return bert_json(BERT_UNCASED)
    if name.startswith("added_"):
        return with_added_tokens(asset_json(name[6:]))
    raise KeyError(name)


def scale_base(name, seed=0, n_corpus=600, n_fuzz=600):
    """base documents of a tiled batch for pipeline `name`: corpus text and fuzz documents (added-token documents for
    added_*), packed -> (data, doc_off)"""
    import corpus
    from fuzzgen import rand_docs
    kind = 4 if name in ("wordpiece", "bert_uncased") else 2
    cd, co = corpus.generate(kind, 300 + seed, 0, n_corpus)
    docs = corpus.to_strings(cd, co)
    if name.startswith("added_"):
        docs += added_token_docs(400 + seed, n_fuzz)
    elif name == "bert_uncased":   # (fuzz documents may hold the combining-mark order the device refuses)
        import random
        rng = random.Random(seed)
        docs += ["".join(chr(0xAC00 + rng.randrange(11172)) for _ in range(rng.randint(1, 40))) + " 中文x ÀÉÎ" for _ in range(n_fuzz // 4)]
    else:
        docs += rand_docs(500 + seed, n_fuzz, max_len=300)
    return pack_docs(docs)


# ---------------------------------------------------------------------------------------------- page-edge placement
PAGE = 2048
EDGES = [0, 32, 256, 416, 1024]
DELTAS = [-40, -33, -32, -31, -17, -16, -9, -8, -4, -3, -2, -1, 0, 1, 2, 3, 4, 8, 9, 16, 17, 31, 32, 33, 40]
FILLER = b"lorem ipsum dolor sit amet, consectetur adipiscing elit "


def place(slots, form, measure=lambda s: len(s.encode("utf-8"))):
    """slots: [(probe, position, anchor)] with position increasing -> documents: the probe's start ("start") or end
    ("end") lands at `position`, counted with `measure` (bytes of the batch the kernels see)"""
    docs, text, pos = [], [], 0
    for probe, p, anchor in slots:
        a = p if anchor == "start" else p - measure(probe)
        gap = a - pos
        assert gap >= 0, (probe, p, anchor)
        fill = (FILLER * (gap // len(FILLER) + 1))[:gap].decode()
        if gap:
            fill = fill[:-1] + "\n"
        if form == "doc":
            docs += [fill, probe]
        else:
            text.append(fill + probe)
            if len(text) == 16:
                docs.append("".join(text)); text = []
        pos = a + measure(probe)
    if text:
        docs.append("".join(text))
    return docs


def page_slots(probes, deltas=DELTAS):
    slots, k = [], 1
    for probe in probes:
        for e in EDGES:
            for anchor in ("start", "end"):
                for d in deltas:
                    slots.append((probe, k * PAGE + e + d, anchor))
                    k += 1
    return slots


def scan_block_slots(probes):
    """around the 2 MiB boundaries of the page and tile scans (1024 pages): one probe per boundary"""
    import random
    rng = random.Random(3)
    out = []
    for m, probe in enumerate(probes, start=1):
        out.append((probe, m * (2 << 20) + rng.choice([-2, -1, 0, 1, 2]), rng.choice(["start", "end"])))
    return out


# probes of the page-edge tests: pre-tokens whose length or content changes the scan's or the model's code path
WIDE = {1: "abcdefghij", 2: "éßжяλ", 3: "中文語あア", 4: "𝒜𝒷𝓬𐐀𐐨"}   # letters (\p{L}) of 1..4 bytes


def word(rng, n_bytes, width):
    """a run of letters of exactly n_bytes, made of `width`-byte characters (ASCII letters first for the remainder)"""
    r = n_bytes % width
    return "".join(rng.choice(WIDE[1]) for _ in range(r)) + "".join(rng.choice(WIDE[width]) for _ in range(n_bytes // width))


def bpe_probes():
    import random
    rng = random.Random(1)
    out = [word(rng, n, w) for n in (16, 17, 24, 25, 32, 33, 255, 256, 257) for w in (1, 2, 3, 4)]
    out += [" " * 40 + "x", "\n" * 33 + "x", " \t" * 20, "x" + " " * 33, "x   \n  y"]          # whitespace runs (\s+(?!\S))
    out += ["don's", "it'S", "we'll", "x''s"]                                              # a contraction split by the edge
    out += ["1" * n for n in (2, 3, 4, 5, 6, 7, 8, 9, 10)]                                 # Llama-3 digit runs of 3k-1, 3k, 3k+1
    out += ["!?!...\r\n\r\nx", "--\r\n", ")]}\r\n\r\n\r\n"]                               # punctuation run + \r\n
    out += ["", "x", "é"]                                                                    # empty and 1-character documents
    return out


def wordpiece_probes(max_chars):
    import random
    rng = random.Random(2)
    out = []
    for n in (max_chars - 1, max_chars, max_chars + 1):
        out += ["".join(rng.choice("abcdefghijklmnop") for _ in range(n)), "".join(rng.choice(WIDE[4]) for _ in range(n))]
    out += ["a" * max_chars, "𝒜" * max_chars, " " * 40 + "x", "x" + "\t" * 33, "don's", "", "x", "é"]
    return out


# characters the BertNormalizer expands: Hangul (three jamo with strip_accents), CJK (spaces around it), accents
BERT_PROBES = ["".join(chr(0xAC00 + (37 * i) % 11172) for i in range(k)) for k in (5, 40, 90)] + ["中文字" * 12, "x中y", "ÀÉÎÕÜ" * 8, "ǅİ"]


_exp = {}


def check(tj, docs, what, wcache=(True, False), byte_offsets=True):
    """the engine against the oracle on `docs` (char offsets, and byte offsets when asked), word cache on and off"""
    from oracle import oracle as orc
    o = orc.Oracle(tj)
    data, off = pack_docs(docs)
    key = (tj, what)
    if key not in _exp:
        _exp[key] = (o.encode_batch_csr(data, off), o.encode_batch_csr(data, off, orc.OFF_BYTE) if byte_offsets else None)
    exp_c, exp_b = _exp[key]
    for wc in wcache:
        tok = tokenizer_with_env(tj, B2T_WCACHE="1" if wc else "0")
        be = tok.encode_batch_csr(data, off)
        assert_csr_equal((be.ids, be.offsets, be.word_ids, be.row_ptr), exp_c, docs, f"{what} wcache={wc}")
        if exp_b is not None:
            be = tok.encode_batch_csr(data, off, byte_offsets=True)
            assert_csr_equal((be.ids, be.offsets, be.word_ids, be.row_ptr), exp_b, docs, f"{what} byte offsets wcache={wc}")


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
