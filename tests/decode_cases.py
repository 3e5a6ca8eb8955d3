"""Shared cases of the decode tests: decoder configurations (tokenizer.json with added tokens), the decoder table as
b2t_decoder_images builds it, a restatement of decode() over that table, and the golden fixture's reader."""
import ctypes, gzip, json, os, random
from types import SimpleNamespace
import numpy as np
import helpers
from tokenizers_b200 import _lib
from tokenizers_b200.tokenizer import parse_tokenizer_json, engine_config, decoder_spec, _char_bytes

BYTELEVEL = {"type": "ByteLevel", "add_prefix_space": True, "trim_offsets": True, "use_regex": True}
WORDPIECE = {"type": "WordPiece", "prefix": "##", "cleanup": True}
# name -> (asset or vocabgen source, decoder)
CONFIGS = {
    "gpt2_bytelevel": ("gpt2_style", BYTELEVEL),
    "llama3_bytelevel": ("llama3_style", BYTELEVEL),
    "wordpiece_cleanup": ("wordpiece", WORDPIECE),
    "wordpiece_no_cleanup": ("wordpiece", dict(WORDPIECE, cleanup=False)),
    "wordpiece_empty_prefix": ("wordpiece", dict(WORDPIECE, prefix="")),
    "wordpiece_no_decoder": ("wordpiece", None),
    "vocabgen_bpe_high": ("vocabgen_bpe", BYTELEVEL),
    "vocabgen_wordpiece_high": ("vocabgen_wordpiece", WORDPIECE),
}
# added tokens: (content, special); "the" is also a vocabulary token, "☃" is outside the byte-level alphabet
ADDED = [("[SPEC]", True), ("<|sp|>", True), ("the", True), ("do not", False), ("' x", False), ("héllo ☃ wörld", False)]


def base_json(src):
    if src == "vocabgen_bpe":
        import vocabgen
        return vocabgen.bpe(5, chain_max=512, vocab_only=(3, 40), id_layout="high")
    if src == "vocabgen_wordpiece":
        import vocabgen
        return vocabgen.wordpiece(5, id_layout="high")
    return helpers.asset_json(src)


def tokenizer_json(name, added=True):
    """the configuration's tokenizer.json, with ADDED at the ids the reference's add_tokens gives them"""
    src, dec = CONFIGS[name]
    j = json.loads(base_json(src))
    j["decoder"] = dec
    if added:
        vocab, toks = j["model"]["vocab"], list(j.get("added_tokens", []))
        # added_vocabulary.rs add_tokens: the model's vocabulary size, or the largest added id + 1 beyond it
        max_added = max([t["id"] for t in toks] + [-1])
        nxt = max_added + 1 if max_added >= len(vocab) else len(vocab)
        for content, special in ADDED:
            if content in vocab:
                tid = vocab[content]
            else:
                tid, nxt = nxt, nxt + 1
            toks.append({"id": tid, "content": content, "single_word": False, "lstrip": False, "rstrip": False,
                         "normalized": not special, "special": special})
        j["added_tokens"] = toks
    return json.dumps(j, ensure_ascii=False)


def added_objects(cfg):
    return [SimpleNamespace(content=t["content"], id=t["id"], special=t.get("special", False),
                            normalized=t.get("normalized", not t.get("special", False))) for t in cfg["added_tokens"] if t.get("content")]


def images(tj, decoder="from_json", normalizer_flags=None, added=None):
    """b2t_decoder_images of a tokenizer.json -> (rc, entries uint64[n_ids], pool uint8)"""
    cfg = parse_tokenizer_json(json.loads(tj))
    if normalizer_flags is not None:
        cfg["normalizer"] = normalizer_flags
    c, keep = engine_config(cfg)
    sp, keep2 = decoder_spec(cfg["decoder"] if decoder == "from_json" else decoder, added if added is not None else added_objects(cfg))
    if sp is None:
        return _lib.B2T_ERR_UNSUPPORTED, None, None
    L = _lib.lib()
    n_ids, nb = ctypes.c_uint32(), ctypes.c_uint64()
    rc = L.b2t_decoder_images(ctypes.byref(c), ctypes.byref(sp), None, None, ctypes.byref(n_ids), ctypes.byref(nb))
    if rc:
        return rc, None, None
    ent, pool = np.zeros(n_ids.value, np.uint64), np.zeros(nb.value, np.uint8)
    _lib.check(L.b2t_decoder_images(ctypes.byref(c), ctypes.byref(sp), ent.ctypes.data, pool.ctypes.data, ctypes.byref(n_ids), ctypes.byref(nb)))
    return rc, ent, pool


def entry(ent, pool, i):
    """-> (exists, skip, first image bytes, later image bytes)"""
    e = int(ent[i])
    off, meta = e & 0xFFFFFFFF, e >> 32
    l1, l2 = meta & 0x3FFF, (meta >> 14) & 0x3FFF
    return bool(meta >> 28 & 1), bool(meta >> 29 & 1), pool[off:off + l1].tobytes(), pool[off + l1:off + l1 + l2].tobytes()


def table_decode(ent, pool, lossy, row, skip):
    """decode() of one row restated over the table: the kernels' algebra in Python"""
    out, first = bytearray(), True
    for i in row:
        i = int(i)
        if i >= ent.size:
            continue
        ex, sk, a, b = entry(ent, pool, i)
        if not ex or (skip and sk):
            continue
        out += a if first else b
        first = False
    return out.decode("utf-8", "replace") if lossy else out.decode("utf-8")


def bytelevel_image(token):
    """the shim's inverse byte map (test_decode_vs_wheel pins it against the reference) for one token"""
    inv = _char_bytes()
    try:
        return bytes(inv[c] for c in token)
    except KeyError:
        return token.encode("utf-8")


def random_rows(seed, n_ids, n_rows, max_len, extra=()):
    """id rows: random ids over [0, n_ids) with a few unknown ones and `extra` ids mixed in"""
    rng = random.Random(seed)
    unknown = [n_ids, n_ids + 1, (1 << 20) - 1, (1 << 20), 0xFFFFFFFF, 0x80000005]
    pool = list(extra) + unknown
    rows = []
    for _ in range(n_rows):
        n = rng.randint(0, max_len)
        rows.append([rng.choice(pool) if rng.random() < 0.08 else rng.randrange(n_ids) for _ in range(n)])
    return rows


def load_golden():
    return json.loads(gzip.open(os.path.join(helpers.GOLDEN, "golden_decode.json.gz")).read().decode("utf-8"))
