"""Deterministic generators of tokenizer.json strings with vocabularies the trained assets never have: tokens up to
512 bytes, ids up to 2^20 - 1, shuffled (non-monotone) merge orders, ignore_merges with vocabulary-only tokens, and
WordPiece with other continuing-subword prefixes and small max_input_chars_per_word.  Test infrastructure, not a test
module; also the targeted documents that drive those vocabularies to their long tokens, and plain restatements of the
facts the engine derives from a vocabulary (monotone merges, soft cuts) so the tests can check their own premises.

Nothing here iterates a set or dict of strings before drawing at random (PYTHONHASHSEED differs between processes)."""
import json
import random

TOP_ID = (1 << 20) - 1          # the highest id the engine accepts (20 id bits in the page kernel)


# ------------------------------------------------------------------------------------------------ byte-level helpers
def _bytes_to_unicode():
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return {b: chr(c) for b, c in zip(bs, cs)}


BYTE_CHAR = _bytes_to_unicode()
CHAR_BYTE = {c: b for b, c in BYTE_CHAR.items()}


def byte_level(s):
    """str (as UTF-8) or bytes -> the ByteLevel string of its bytes"""
    if isinstance(s, str):
        s = s.encode("utf-8")
    return "".join(BYTE_CHAR[b] for b in s)


def from_byte_level(s):
    """a ByteLevel token string -> its bytes, or None when it holds a character outside the ByteLevel alphabet"""
    try:
        return bytes(CHAR_BYTE[c] for c in s)
    except KeyError:
        return None


# ------------------------------------------------------------------------------------------------ restatements
def is_monotone(vocab, merges):
    """True iff every merge ranks after every merge that creates one of its parts (rank = position in `merges`; a later
    duplicate of a pair replaces the earlier one, and any duplicate makes the table count as not monotone).
    vocab: token string -> id; merges: [(a, b)] token strings."""
    table = {}
    for r, (a, b) in enumerate(merges):
        table[(vocab[a], vocab[b])] = (r, vocab[a + b])
    if len(table) != len(merges):
        return False
    created = {}
    for r, new in table.values():
        created[new] = max(created.get(new, -1), r)
    return all(created.get(x, -1) < r and created.get(y, -1) < r for (x, y), (r, _) in table.items())


def soft_cuts(tokens, raw):
    """raw bytes of one pre-token -> its pieces: a cut before byte i wherever no token can hold bytes i-1 and i side by
    side (the pair is not a token, and neither byte triple around the boundary occurs inside a token).
    tokens: iterable of token byte strings."""
    pairs, triples = set(), set()
    for t in tokens:
        if len(t) == 2:
            pairs.add(t)
        for p in range(len(t) - 2):
            triples.add(t[p:p + 3])
    pieces, a = [], 0
    for i in range(1, len(raw)):
        if raw[i - 1:i + 1] in pairs:
            continue
        if i >= 2 and raw[i - 2:i + 1] in triples:
            continue
        if i + 1 < len(raw) and raw[i - 1:i + 2] in triples:
            continue
        pieces.append(raw[a:i])
        a = i
    pieces.append(raw[a:])
    return pieces


# ------------------------------------------------------------------------------------------------ BPE
RANDOM_ALPHABET = "etoinshrdlucmfwyp.,!'0123456789é"   # random merges: no chain letter, nothing of QRSTUV
VOCAB_ONLY_ALPHABET = "WXYZKLMNOPGHJ"                  # letters no merge touches
PIECE_TOKEN = "QRSTUV"                                 # vocabulary-only, and a soft-cut piece of PIECE_RUN
PIECE_RUN = "QRSTUV!" * 60 + "QRSTUV"                  # 426 bytes, cut around every "!"
PRETOKENIZERS = {
    "gpt2": {"type": "ByteLevel", "add_prefix_space": False, "trim_offsets": True, "use_regex": True},
    "noregex": {"type": "ByteLevel", "add_prefix_space": False, "trim_offsets": True, "use_regex": False},
    "prefix": {"type": "ByteLevel", "add_prefix_space": True, "trim_offsets": True, "use_regex": True},
    "llama3": {"type": "Sequence", "pretokenizers": [
        {"type": "Split", "pattern": {"Regex": "(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\\r\\n\\p{L}\\p{N}]?\\p{L}+|\\p{N}{1,3}| ?[^\\s\\p{L}\\p{N}]+[\\r\\n]*|\\s*[\\r\\n]+|\\s+(?!\\S)|\\s+"},
         "behavior": "Isolated", "invert": False},
        {"type": "ByteLevel", "add_prefix_space": False, "trim_offsets": True, "use_regex": False}]},
}


def ltr_word(seed, n):
    """the left-to-right chain's word: n letters outside the chains, whose first letter pair occurs only at its start
    (so every prefix of it merges into one token)"""
    rng = random.Random(seed * 7919 + 1)
    letters = "cdefghijklmnopqrstuvwxyz"
    w = [rng.choice(letters), rng.choice(letters)]
    while len(w) < n:
        c = rng.choice(letters)
        if not (w[-1] == w[0] and c == w[1]):
            w.append(c)
    return "".join(w)


def vocab_only_tokens(seed, sizes):
    """tokens no merge produces: PIECE_TOKEN for size 6, else `size` letters of VOCAB_ONLY_ALPHABET"""
    rng = random.Random(seed * 104729 + 3)
    return [PIECE_TOKEN if n == 6 else "".join(rng.choice(VOCAB_ONLY_ALPHABET) for _ in range(n)) for n in sizes]


def _assign_ids(rng, tokens, layout, spread, top_token=None):
    """token list -> {token: id}: dense from 0 in list order, or ("high") scattered in [2^20 - spread V, 2^20) with
    TOP_ID given to `top_token` (the first token when None)"""
    if layout == "dense":
        return {t: i for i, t in enumerate(tokens)}
    V = len(tokens)
    ids = rng.sample(range((1 << 20) - spread * V, TOP_ID), V - 1)
    top = tokens.index(top_token) if top_token is not None else 0
    ids.insert(top, TOP_ID)
    return dict(zip(tokens, ids))


def bpe(seed, chains="ab ", chain_max=512, ltr=300, n_random=300, shuffle=False, ignore_merges=False, vocab_only=(),
        id_layout="dense", spread=4, pretok="gpt2"):
    """Byte-level BPE.  Merges, in this order: doubling chains c, cc, c^4 .. c^chain_max for each c in `chains`; a
    left-to-right chain w[:1] + w[1], .. w[:ltr-1] + w[ltr-1] of ltr_word(seed, ltr) (tokens of every length 2..ltr);
    n_random merges of two existing tokens over RANDOM_ALPHABET.  `shuffle` permutes the merges (not monotone any
    more).  `vocab_only`: sizes of vocab_only_tokens(seed, ...), in the vocabulary but produced by no merge.
    Byte "a" takes TOP_ID under id_layout="high"."""
    rng = random.Random(seed)
    toks = [bytes([b]) for b in range(256)]
    known = set(toks)
    merges = []

    def merge(a, b):
        merges.append((a, b))
        if a + b not in known:
            known.add(a + b)
            toks.append(a + b)

    for c in chains:
        t = c.encode()
        while 2 * len(t) <= chain_max:
            merge(t, t)
            t += t
    if ltr:
        w = ltr_word(seed, ltr).encode()
        for k in range(1, ltr):
            merge(w[:k], w[k:k + 1])
    pool = [bytes([b]) for b in sorted(set(RANDOM_ALPHABET.encode()))]
    for _ in range(n_random):
        for _attempt in range(20):
            a, b = rng.choice(pool), rng.choice(pool)
            if a + b not in known and len(a + b) <= 48:
                merge(a, b)
                pool.append(a + b)
                break
    if shuffle:
        rng.shuffle(merges)
    extra = [t.encode() for t in vocab_only_tokens(seed, vocab_only)]
    assert not any(t in known for t in extra)
    strings = [byte_level(t) for t in toks + extra]
    vocab = _assign_ids(rng, strings, id_layout, spread, byte_level("a"))
    model = {"type": "BPE", "dropout": None, "unk_token": None, "continuing_subword_prefix": None, "end_of_word_suffix": None,
             "fuse_unk": False, "byte_fallback": False, "ignore_merges": bool(ignore_merges), "vocab": vocab,
             "merges": [[byte_level(a), byte_level(b)] for a, b in merges]}
    return json.dumps({"version": "1.0", "truncation": None, "padding": None, "added_tokens": [], "normalizer": None,
                       "pre_tokenizer": PRETOKENIZERS[pretok], "post_processor": None, "decoder": None, "model": model},
                      ensure_ascii=False)


# ------------------------------------------------------------------------------------------------ WordPiece
WP_LETTERS = "abcdefgh" + "жяλß" + "あいうえ" + "𝒷𝓬𝒹𐐨"   # 1- to 4-byte letters, lowercase (stable under BertNormalizer)
WP_WIDE = "𝒷𝓬𝒹𐐨"
WP_NO_CONT = "h"          # a whole token, never a continuing piece: a word with it inside fails to match
WP_MISSING = "z"          # in no token: a word with it fails to match


def wordpiece(seed, prefix="##", max_chars=100, unk_id=None, n_stems=300, long_sizes=(24, 50, 100, 104), id_layout="dense",
              spread=4, pretok="whitespace"):
    """WordPiece over WP_LETTERS.  Stems of 2..8 letters, each with some of its proper prefixes (gaps force the
    longest match to fall back) and continuing forms `prefix` + stem and + some of its prefixes; every letter whole and
    (except WP_NO_CONT) continuing; stems of WP_WIDE letters of `long_sizes` characters; [UNK] in the middle, with id
    `unk_id` when given (dense layout; the "high" layout gives it TOP_ID).  pretok: "whitespace" (Whitespace) or "bert" (BertNormalizer uncased + BertPreTokenizer)."""
    rng = random.Random(seed)
    toks = []
    seen = set()

    def add(t):
        if t not in seen:
            seen.add(t)
            toks.append(t)

    for c in WP_LETTERS:
        add(c)
        if c != WP_NO_CONT:
            add(prefix + c)
    add(WP_NO_CONT)
    for _ in range(n_stems):
        stem = "".join(rng.choice(WP_LETTERS) for _ in range(rng.randint(2, 8)))
        for k in range(2, len(stem)):
            if rng.random() < 0.5:
                add(stem[:k])
        add(stem)
        if rng.random() < 0.5:
            for k in range(2, len(stem)):
                if rng.random() < 0.3:
                    add(prefix + stem[:k])
            add(prefix + stem)
    for n in long_sizes:
        stem = "".join(rng.choice(WP_WIDE) for _ in range(n))
        add(stem)
        add(prefix + stem[1:])
    toks.insert(len(toks) // 2, "[UNK]")
    vocab = _assign_ids(rng, toks, id_layout, spread, "[UNK]")
    if unk_id is not None and id_layout == "dense":
        vocab = {t: (unk_id if t == "[UNK]" else i) for t, i in vocab.items()}
    if pretok == "bert":
        nz = {"type": "BertNormalizer", "clean_text": True, "handle_chinese_chars": True, "strip_accents": None, "lowercase": True}
        pt = {"type": "BertPreTokenizer"}
    else:
        nz, pt = None, {"type": "Whitespace"}
    model = {"type": "WordPiece", "unk_token": "[UNK]", "continuing_subword_prefix": prefix, "max_input_chars_per_word": max_chars,
             "vocab": vocab}
    return json.dumps({"version": "1.0", "truncation": None, "padding": None, "added_tokens": [], "normalizer": nz,
                       "pre_tokenizer": pt, "post_processor": None, "decoder": None, "model": model}, ensure_ascii=False)


# ------------------------------------------------------------------------------------------------ configurations
class Config:
    """a named generator call and what it claims: `monotone` (BPE), the highest id, the longest token in bytes"""

    def __init__(self, name, gen, kwargs, max_id, longest, monotone=None):
        self.name, self.gen, self.kwargs = name, gen, kwargs
        self.max_id, self.longest, self.monotone = max_id, longest, monotone

    @property
    def kind(self):
        return "bpe" if self.gen is bpe else "wordpiece"

    def json(self):
        return self.gen(**self.kwargs)

    def __repr__(self):
        return self.name


VOCAB_ONLY_SIZES = (6, 40, 100, 256, 300)

CONFIGS = [
    Config("bpe_gpt2", bpe, dict(seed=1), max_id=None, longest=512, monotone=True),
    Config("bpe_noregex_high", bpe, dict(seed=2, id_layout="high", pretok="noregex"), max_id=TOP_ID, longest=512, monotone=True),
    Config("bpe_prefix_shuffled", bpe, dict(seed=3, shuffle=True, id_layout="high", pretok="prefix"), max_id=TOP_ID, longest=512, monotone=False),
    Config("bpe_noregex_shuffled", bpe, dict(seed=4, shuffle=True, id_layout="high", spread=2, pretok="noregex", n_random=150),
           max_id=TOP_ID, longest=512, monotone=False),
    Config("bpe_llama3_ignore", bpe, dict(seed=5, ignore_merges=True, vocab_only=VOCAB_ONLY_SIZES, id_layout="high", pretok="llama3"),
           max_id=TOP_ID, longest=512, monotone=True),
    Config("bpe_gpt2_ignore", bpe, dict(seed=6, ignore_merges=True, vocab_only=VOCAB_ONLY_SIZES, id_layout="high"),
           max_id=TOP_ID, longest=512, monotone=True),
    Config("bpe_noregex_ignore", bpe, dict(seed=7, ignore_merges=True, vocab_only=VOCAB_ONLY_SIZES, id_layout="high", pretok="noregex"),
           max_id=TOP_ID, longest=512, monotone=True),
    Config("wp_hash_104", wordpiece, dict(seed=11, prefix="##", max_chars=104, id_layout="high"), max_id=TOP_ID, longest=416),
    Config("wp_empty_5", wordpiece, dict(seed=12, prefix="", max_chars=5, unk_id=TOP_ID), max_id=TOP_ID, longest=416),
    Config("wp_sp_24_bert", wordpiece, dict(seed=13, prefix="▁", max_chars=24, id_layout="high", pretok="bert"), max_id=TOP_ID, longest=416),
    Config("wp_atat_1", wordpiece, dict(seed=14, prefix="@@", max_chars=1, unk_id=TOP_ID), max_id=TOP_ID, longest=416),
    Config("wp_hash_100_bert", wordpiece, dict(seed=15, prefix="##", max_chars=100, pretok="bert"), max_id=None, longest=416),
]
BY_NAME = {c.name: c for c in CONFIGS}


# ------------------------------------------------------------------------------------------------ targeted documents
RUN_LENGTHS = (1, 2, 3, 15, 16, 17, 23, 24, 25, 31, 32, 33, 63, 64, 65, 255, 256, 257, 511, 512, 513, 1024, 2100)
LTR_PREFIXES = (24, 32, 33, 256, 257, 300)


def _utf8_tokens(tj):
    """the vocabulary's tokens that are whole UTF-8 text, in id order"""
    v = json.loads(tj)["model"]["vocab"]
    out = []
    for t, _ in sorted(v.items(), key=lambda kv: kv[1]):
        raw = from_byte_level(t)
        try:
            out.append(raw.decode("utf-8"))
        except (AttributeError, UnicodeDecodeError):
            pass
    return out


def bpe_probes(cfg):
    """documents of a BPE configuration that reach its long tokens: chain runs (alone, and with a letter after the
    space runs), prefixes of the left-to-right word, the vocabulary-only tokens (alone and in context), the piece
    construction, and concatenations of random vocabulary tokens"""
    kw = cfg.kwargs
    seed = kw["seed"]
    rng = random.Random(seed + 1000)
    out = []
    for c in kw.get("chains", "ab "):
        for n in RUN_LENGTHS:
            out.append(c * n)
            if c == " ":
                out.append(c * n + "x")
    w = ltr_word(seed, kw.get("ltr", 300))
    out += [w[:k] for k in LTR_PREFIXES if k <= len(w)]
    out += ["x " + w[:k] + "!" for k in (33, 257)]
    for t in vocab_only_tokens(seed, kw.get("vocab_only", ())):
        out += [t, "x\n" + t, t + "!", " " + t, t[:-1], t + t]
        if len(t) <= 256:   # one pre-token of more than 256 bytes without regex, soft-cut into copies of t
            out.append("!".join([t] * (1 + 300 // len(t))))
    out += [PIECE_RUN, PIECE_TOKEN, PIECE_TOKEN + "!" + PIECE_TOKEN, "!" + PIECE_RUN + "!"]
    toks = _utf8_tokens(cfg.json())
    long_toks = [t for t in toks if len(t.encode()) > 16]
    for _ in range(40):
        parts = [rng.choice(long_toks if rng.random() < 0.5 else toks) for _ in range(rng.randint(1, 8))]
        out.append("".join(parts))
    return out


def abc_word(n):
    """n letters that always match (each is a token whole and continuing): [UNK] only past max_input_chars_per_word"""
    return "".join("abcdefg"[i % 7] for i in range(n))


def wordpiece_probes(cfg):
    """documents of a WordPiece configuration: words of max_chars - 1, max_chars and max_chars + 1 characters (1-byte
    and 4-byte letters), words that make the longest match fall back or fail, words made of continuing pieces only,
    and words of WP_WIDE letters up to 104 characters (the whole 416-byte halo)"""
    kw = cfg.kwargs
    rng = random.Random(kw["seed"] + 2000)
    m = kw.get("max_chars", 100)
    prefix = kw.get("prefix", "##")
    v = json.loads(cfg.json())["model"]["vocab"]
    toks = sorted(v, key=lambda t: v[t])
    whole = [t for t in toks if t != "[UNK]" and (not prefix or not t.startswith(prefix))]
    cont = [t[len(prefix):] for t in toks if prefix and t.startswith(prefix) and len(t) > len(prefix)] or whole
    out = []
    for n in (m - 1, m, m + 1):
        if n > 0:
            out += [abc_word(n), "".join(rng.choice("abcdefg") for _ in range(n)), "".join(rng.choice(WP_WIDE) for _ in range(n))]
    for _ in range(30):   # a whole token, then continuing pieces: the longest match has to step back over the gaps
        out.append(rng.choice(whole) + "".join(rng.choice(cont) for _ in range(rng.randint(1, 3))))
    for _ in range(15):   # continuing pieces only
        out.append("".join(rng.choice(cont) for _ in range(rng.randint(1, 4))))
    short = [t for t in whole if len(t) <= 4]
    out += ["a" + WP_NO_CONT, rng.choice(short) + WP_NO_CONT + rng.choice(short), WP_MISSING, "ab" + WP_MISSING, WP_MISSING + "ab"]
    for n in (24, 50, 99, 100, 103, 104, 105):
        out.append("".join(rng.choice(WP_WIDE) for _ in range(n)))
    out += [" ".join(rng.choice(short) for _ in range(12)) for _ in range(5)]
    return out


def probes(cfg):
    return bpe_probes(cfg) if cfg.kind == "bpe" else wordpiece_probes(cfg)


def fuzz_docs(cfg, n):
    from fuzzgen import rand_docs
    return rand_docs(3000 + cfg.kwargs["seed"], n, max_len=60)
