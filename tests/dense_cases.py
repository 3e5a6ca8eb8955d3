"""TEST INFRASTRUCTURE: what the dense-mode tests (test_dense*.py) and their golden maker (golden/make_golden_dense.py)
share -- the tokenizers, the settings and inputs of each mode, the reference wheel's rows, the committed fixtures, the one
comparison of rows or errors, and the host build of the row kernels (native/dense_emul.cpp) with its runner."""
import ctypes, gzip, json, os, random, subprocess
import numpy as np
import pytest
import helpers, fuzzgen, corpus
import dense_oracle
from tokenizers_b200.tokenizer import parse_post_processor, special_token_count

tk = helpers.wheel()
HERE = os.path.dirname(os.path.abspath(__file__))
STRATEGIES = ("longest_first", "only_first", "only_second")
TOO_SHORT = "Truncation error: Sequence to truncate too short to respect the provided max_length"
PANIC = "must be strictly less than `max_len"
NOT_FIT = "does not fit"
WORDS = ["the", "cat", "sat", "on", "a", "mat", "why", "not", "blue", "run"]


# ------------------------------------------------------------------------------------------------- tokenizers
def _gpt2_template(v):
    return {"type": "TemplateProcessing",
            "single": [{"SpecialToken": {"id": "<s>", "type_id": 0}}, {"Sequence": {"id": "A", "type_id": 0}},
                       {"SpecialToken": {"id": "</s>", "type_id": 0}}, {"SpecialToken": {"id": "<s>", "type_id": 0}}],
            "pair": [{"Sequence": {"id": "A", "type_id": 0}}, {"Sequence": {"id": "B", "type_id": 1}}],
            "special_tokens": {"<s>": {"id": "<s>", "ids": [v["a"]], "tokens": ["a"]},
                               "</s>": {"id": "</s>", "ids": [v["b"], v["c"]], "tokens": ["b", "c"]}}}


def _bert(v):
    return {"type": "BertProcessing", "sep": ["[SEP]", v["[SEP]"]], "cls": ["[CLS]", v["[CLS]"]]}


def _template_b_first(v):
    """TemplateProcessing with B before A, a special token of two ids and type ids 0 / 1 / 2"""
    return {"type": "TemplateProcessing",
            "single": [{"SpecialToken": {"id": "[CLS]", "type_id": 2}}, {"Sequence": {"id": "A", "type_id": 0}}],
            "pair": [{"SpecialToken": {"id": "[CLS]", "type_id": 2}}, {"Sequence": {"id": "B", "type_id": 1}},
                     {"SpecialToken": {"id": "<two>", "type_id": 0}}, {"Sequence": {"id": "A", "type_id": 0}},
                     {"SpecialToken": {"id": "[CLS]", "type_id": 2}}],
            "special_tokens": {"[CLS]": {"id": "[CLS]", "ids": [v["[CLS]"]], "tokens": ["[CLS]"]},
                               "<two>": {"id": "<two>", "ids": [v["[SEP]"], v["[MASK]"]], "tokens": ["[SEP]", "[MASK]"]}}}


def _roberta(aps):
    return lambda v: {"type": "RobertaProcessing", "sep": ["b", v["b"]], "cls": ["a", v["a"]], "trim_offsets": True, "add_prefix_space": aps}


def _bytelevel(v):
    return {"type": "ByteLevel", "add_prefix_space": True, "trim_offsets": True, "use_regex": True}


def _seq_bytelevel_template(v):
    """Sequence[ByteLevel(trim_offsets, add_prefix_space false), TemplateProcessing]"""
    return {"type": "Sequence", "processors": [
        {"type": "ByteLevel", "add_prefix_space": False, "trim_offsets": True, "use_regex": True},
        {"type": "TemplateProcessing",
         "single": [{"SpecialToken": {"id": "a", "type_id": 0}}, {"Sequence": {"id": "A", "type_id": 0}}, {"SpecialToken": {"id": "b", "type_id": 0}}],
         "pair": [{"SpecialToken": {"id": "a", "type_id": 0}}, {"Sequence": {"id": "A", "type_id": 0}}, {"SpecialToken": {"id": "b", "type_id": 0}},
                  {"Sequence": {"id": "B", "type_id": 1}}, {"SpecialToken": {"id": "b", "type_id": 1}}],
         "special_tokens": {"a": {"id": "a", "ids": [v["a"]], "tokens": ["a"]}, "b": {"id": "b", "ids": [v["b"]], "tokens": ["b"]}}}]}


# added tokens of the `roberta_added` tokenizer: (content, single_word, lstrip, rstrip, normalized, special)
ADDED_SPECS = [("<mask>", False, True, False, False, True), ("[SEP2]", False, False, True, False, True),
               ("<both>", False, True, True, False, True), ("<|endoftext|>", False, False, False, False, True)]

# name -> (asset, post-processor from the vocabulary, pre-tokenizer add_prefix_space, added tokens)
TEMPLATES = {
    "gpt2_style": ("gpt2_style", _gpt2_template, False, False),
    "wordpiece": ("wordpiece", _bert, False, False),
    "llama3_style": ("llama3_style", lambda v: None, False, False),
    "bert": ("wordpiece", _bert, False, False),
    "roberta": ("gpt2_style", _roberta(False), False, False),
    "b_first": ("wordpiece", _template_b_first, False, False),
    "none": ("llama3_style", lambda v: None, False, False),
    "roberta_aps": ("gpt2_style", _roberta(True), False, False),
    "bytelevel": ("gpt2_style", _bytelevel, False, False),
    "seq_template": ("llama3_style", _seq_bytelevel_template, False, False),
    "gpt2_prefix": ("gpt2_style", _bytelevel, True, False),
    "roberta_added": ("gpt2_style", _roberta(True), False, True),
}


def tokenizer_json(name):
    asset, pp, prefix, added = TEMPLATES[name]
    js = json.loads(helpers.asset_json(asset))
    js["post_processor"] = pp(js["model"]["vocab"])
    if prefix:
        js["pre_tokenizer"] = dict(js["pre_tokenizer"], add_prefix_space=True)
    if added:
        js["added_tokens"] = helpers.added_token_entries(js["model"]["vocab"], ADDED_SPECS)
    return json.dumps(js)


# ------------------------------------------------------------------------------- single sequences (test_dense)
DENSE_NAMES = ["gpt2_style", "wordpiece", "llama3_style"]
# (truncation | None, padding)
DENSE_SETTINGS = [
    (dict(max_length=16, direction="right"), dict(length=16, direction="right", pad_id=0)),
    (dict(max_length=12, direction="left"), dict(length=None, direction="left", pad_id=3)),
    (dict(max_length=40, direction="right"), dict(length=None, direction="right", pad_id=1, pad_to_multiple_of=8)),
    (None, dict(length=None, direction="right", pad_id=2)),
    (dict(max_length=7, direction="right"), dict(length=20, direction="left", pad_id=5, pad_to_multiple_of=16)),
]


def docs_for(seed):
    return fuzzgen.rand_docs(seed, 600, max_len=120) + ["", " ", "a", "hello world " * 30]


# ------------------------------------------------------------------------------------------ pairs (test_dense_pairs)
PAIR_NAMES = ["bert", "roberta", "b_first", "none"]
# (truncation | None, padding); max_length "special" = exactly the special tokens of the template: a budget of 0
PAIR_SETTINGS = [
    (dict(max_length=40, strategy="longest_first", direction="right"), dict(length=40, direction="right", pad_id=0, pad_type_id=0)),
    (dict(max_length=33, strategy="longest_first", direction="left"), dict(length=None, direction="left", pad_id=3, pad_type_id=1)),
    (dict(max_length=30, strategy="only_first", direction="right"), dict(length=None, direction="right", pad_id=1, pad_type_id=2, pad_to_multiple_of=8)),
    (dict(max_length=24, strategy="only_second", direction="left"), dict(length=40, direction="left", pad_id=5, pad_type_id=0, pad_to_multiple_of=16)),
    (dict(max_length=40, strategy="only_first", direction="left"), dict(length=None, direction="right", pad_id=2, pad_type_id=7)),
    (dict(max_length=36, strategy="only_second", direction="right"), dict(length=None, direction="left", pad_id=2, pad_type_id=0)),
    (None, dict(length=None, direction="right", pad_id=2, pad_type_id=0)),
    (dict(max_length="special", strategy="only_first", direction="right"), dict(length=None, direction="right", pad_id=9, pad_type_id=3)),
]
# pairs with a cut the strategy cannot make: SequenceTooShort (B alone fills the budget / A alone does / A would go to 0)
ERROR_CASES = [
    ("hello", "the second sequence is much longer than this budget " * 2, dict(max_length=16, strategy="only_first", direction="right")),
    ("the first sequence is much longer than this budget " * 2, "hi", dict(max_length=16, strategy="only_second", direction="left")),
]


def pair_cases():
    for k, (tr, pd) in enumerate(PAIR_SETTINGS):
        for ast in (True, False):
            yield f"{k}/{int(ast)}", tr, pd, ast


def pairs_for(seed, n=150):
    """(fuzz document, short sentence of at most four words) pairs, and the empty corner cases"""
    rng = random.Random(seed)
    long_ = fuzzgen.rand_docs(seed, n, max_len=90)
    short = [" ".join(rng.choice(WORDS) for _ in range(rng.randint(0, 4))) for _ in range(n)]
    return list(zip(long_, short)) + [("", ""), ("a", ""), ("", "b"), ("hello world " * 8, "x")]


# ------------------------------------------------------------------------ overflowing parts (test_dense_overflow)
# (truncation, padding).  stride "b-1": the budget (max_length less the template's special tokens) - 1, where every cut
# sequence panics under only_first / only_second (its max_len is below the budget) and longest_first panics on some pairs.
OVERFLOW_SETTINGS = [
    (dict(max_length=24, stride=0, strategy="longest_first", direction="right"), dict(length=24, direction="right", pad_id=0, pad_type_id=0)),
    (dict(max_length=20, stride=1, strategy="only_second", direction="left"), dict(length=None, direction="left", pad_id=3, pad_type_id=1, pad_to_multiple_of=8)),
    (dict(max_length=28, stride=5, strategy="only_first", direction="right"), dict(length=None, direction="right", pad_id=1, pad_type_id=2)),
    (dict(max_length=30, stride=4, strategy="longest_first", direction="left"), dict(length=32, direction="right", pad_id=2, pad_type_id=0)),
    (dict(max_length=26, stride="b-1", strategy="only_second", direction="right"), dict(length=None, direction="right", pad_id=2, pad_type_id=0)),
    (dict(max_length=26, stride="b-1", strategy="longest_first", direction="right"), dict(length=None, direction="right", pad_id=2, pad_type_id=0)),
]


def overflow_cases():
    for k, (tr, pd) in enumerate(OVERFLOW_SETTINGS):
        for is_pair in (True, False):
            if not is_pair and tr["strategy"] == "only_second":
                continue   # (a single sequence has no second one to cut: the reference refuses)
            for ast in (True, False):
                yield f"{k}/{'pair' if is_pair else 'single'}/{int(ast)}", tr, pd, is_pair, ast


def overflow_inputs(seed, n=60):
    """pairs of a fuzz document and a short sentence, long contexts that make many windows, and the empty corner cases"""
    ps = pairs_for(seed, n)
    rng = random.Random(seed)
    long_ = [" ".join(rng.choice(WORDS) for _ in range(rng.randint(40, 120))) for _ in range(4)]
    return ps + [(t, "why not") for t in long_]


def qa_inputs():
    """questions with corpus contexts: pairs around 64 KiB chunk edges, a context larger than a chunk (hundreds of
    windows), and enough windows in all to grow the pinned rows past their first guess (one row per input)"""
    data, off = corpus.generate(2, 33, 0, 600)
    docs = corpus.to_strings(data, off)
    qs = ["what is " + " ".join(d.split()[:3]) for d in docs]
    ps = list(zip(qs, docs))
    filler = "lorem ipsum dolor sit amet, consectetur adipiscing elit "
    ps.append(("where is the end?", (filler * 2000)[:90000]))
    return ps + list(zip(qs[::-1], docs[::-1]))[:100]


# ----------------------------------------------------------------------------------- row metadata (test_dense_meta)
META_NAMES = ["roberta", "roberta_aps", "bytelevel", "seq_template", "gpt2_prefix", "roberta_added", "bert", "b_first", "none"]
# (truncation | None, padding, return_overflowing_tokens)
META_SETTINGS = [
    (dict(max_length=16, stride=3, strategy="longest_first", direction="right"), dict(length=24, direction="right", pad_id=0, pad_type_id=0), True),
    (dict(max_length=32, stride=1, strategy="only_second", direction="left"), dict(length=None, direction="left", pad_id=3, pad_type_id=1, pad_to_multiple_of=8), True),
    (dict(max_length=14, stride=0, strategy="longest_first", direction="left"), dict(length=None, direction="right", pad_id=2, pad_type_id=0), False),
    (None, dict(length=None, direction="right", pad_id=1, pad_type_id=2), False),
]


def meta_cases():
    for k, (tr, pd, over) in enumerate(META_SETTINGS):
        for is_pair in (True, False):
            if not is_pair and tr is not None and tr["strategy"] == "only_second":
                continue
            for ast in (True, False):
                yield f"{k}/{'pair' if is_pair else 'single'}/{int(ast)}", tr, pd, over, is_pair, ast


WS_DOCS = ["hello  there world of cats", "and dogs  too", "a\n\n  b   c", "  leading spaces", "trailing spaces   ", "tab\t\tsep  x",
           "  ", "", "one", "x  y  z  w  v  u  t  s  r  q  p  o", "why   not  blue    run the cat sat on a mat"]
ADDED_DOCS = ["cat  <mask>", "cat<mask> dog", "the <mask> sat", "x　 <mask> y", "a [SEP2]  b", "a [SEP2]b", "[SEP2]\t\tz",
              "q<both>r", "<both>!", "<|endoftext|>  hi", "  <mask>  [SEP2]  x", "no added tokens here  at all"]


def meta_inputs(name, seed, n=24):
    """pairs of documents with whitespace runs and short sentences; for the added-token tokenizer, documents with added
    tokens that absorbed 0, 1 and several whitespace chars (<both> absorbing none)"""
    rng = random.Random(seed)
    docs = ADDED_DOCS if name == "roberta_added" else WS_DOCS
    ps = [(rng.choice(docs) + " " + " ".join(rng.choice(WORDS) + " " * rng.randint(1, 3) for _ in range(rng.randint(0, 8))),
           rng.choice(docs)) for _ in range(n)]
    return [("hello  there world of cats", "and dogs  too")] + ps + [(d, e) for d, e in zip(docs, docs[1:])]


# ------------------------------------------------------------------------------------------------------ settings
def arrange(seqs, tr, is_pair=True):
    """the inputs a setting runs on: single sequences take the first of each pair; pairs the short sentence second for
    only_first and first for only_second (so that the strategy's sequence can always be cut), alternating otherwise (so
    that longest_first sees both orders)"""
    if not is_pair:
        return [a for a, _ in seqs]
    if tr is not None and tr["strategy"] == "only_first":
        return seqs
    if tr is not None and tr["strategy"] == "only_second":
        return [(b, a) for a, b in seqs]
    return [(a, b) if k % 2 else (b, a) for k, (a, b) in enumerate(seqs)]


def n_special(js, is_pair=True):
    return special_token_count(parse_post_processor(json.loads(js).get("post_processor")), is_pair)


def resolve(js, tr, is_pair=True, ast=True):
    """the setting with max_length "special" resolved to the special tokens of the pair template (None where that has no
    dense form: max_length 0), and stride "b-1" against the template's budget (the reference's enable_truncation refuses a
    stride that is not below max_length less the special tokens of a single sequence)"""
    if tr is not None and tr["max_length"] == "special":
        m = n_special(js)
        return dict(tr, max_length=m) if m else None
    if tr is not None and tr.get("stride") == "b-1":
        budget = tr["max_length"] - (n_special(js, is_pair) if ast else 0)
        return dict(tr, stride=max(min(budget, tr["max_length"] - n_special(js, False)) - 1, 0))
    return tr


def flat(x):
    return [s for p in x for s in (p if isinstance(p, (tuple, list)) else (p,))]


def apply(tok, tr, pd):
    """the setting on a tokenizer (the shim's or the wheel's)"""
    tok.no_truncation(); tok.no_padding()
    if tr:
        tok.enable_truncation(tr["max_length"], stride=tr.get("stride", 0), strategy=tr.get("strategy", "longest_first"), direction=tr["direction"])
    tok.enable_padding(direction=pd["direction"], pad_id=pd["pad_id"], pad_type_id=pd.get("pad_type_id", 0), length=pd["length"],
                       pad_to_multiple_of=pd.get("pad_to_multiple_of"))


# ------------------------------------------------------------------------------------------------ rows and errors
FIELDS = ("ids", "type_ids", "mask", "lengths", "sample", "offsets", "special_tokens_mask", "sequence_ids", "word_ids")
GOLDEN_KEYS = ("ids", "type_ids", "mask", "lengths", "sample", "offsets", "special", "seq", "words")
DTYPES = (np.uint32, np.uint8, np.uint8, np.uint32, np.uint32, np.uint32, np.uint8, np.int8, np.int32)


def wheel_rows(js, inputs, tr, pd, ast=True, over=False):
    """the reference: encode_batch with truncation and padding, every input's Encoding (and with `over` its overflowing
    Encodings) stacked in that order -> the nine FIELDS, or the error message"""
    tok = tk.Tokenizer.from_str(js)
    apply(tok, tr, pd)
    try:
        encs = tok.encode_batch(inputs, add_special_tokens=ast)
    except BaseException as ex:   # (the stride check is a Rust panic: PanicException derives from BaseException)
        if isinstance(ex, (KeyboardInterrupt, SystemExit)):
            raise
        return str(ex)
    rows, sample = [], []
    for p, e in enumerate(encs):
        for x in [e] + (list(e.overflowing) if over else []):
            rows.append(x); sample.append(p)
    widths = {len(x.ids) for x in rows}
    if len(widths) > 1:
        return f"rows of {sorted(widths)} tokens: a row does not fit L"
    R, L = len(rows), widths.pop() if widths else 0
    none = lambda v: -1 if v is None else v
    return (np.array([x.ids for x in rows], dtype=np.uint32).reshape(R, L), np.array([x.type_ids for x in rows], dtype=np.uint8).reshape(R, L),
            np.array([x.attention_mask for x in rows], dtype=np.uint8).reshape(R, L), np.array([sum(x.attention_mask) for x in rows], dtype=np.uint32),
            np.array(sample, dtype=np.uint32), np.array([x.offsets for x in rows], dtype=np.uint32).reshape(R, L, 2),
            np.array([x.special_tokens_mask for x in rows], dtype=np.uint8).reshape(R, L),
            np.array([[none(s) for s in x.sequence_ids] for x in rows], dtype=np.int8).reshape(R, L),
            np.array([[none(w) for w in x.word_ids] for x in rows], dtype=np.int32).reshape(R, L))


def golden(name):
    """the committed fixture tests/golden/golden_<name>.json.gz"""
    return json.loads(gzip.open(os.path.join(helpers.GOLDEN, f"golden_{name}.json.gz")).read().decode("utf-8"))


def golden_rows(c):
    """a fixture record -> the nine FIELDS, None where the record has none, or its error message"""
    if "error" in c:
        return c["error"]
    R, L = c["shape"]
    shapes = {"lengths": (R,), "sample": (R,), "offsets": (R, L, 2)}
    return tuple(np.array(c[k], dtype=dt).reshape(shapes.get(nm, (R, L))) if k in c else None for nm, k, dt in zip(FIELDS, GOLDEN_KEYS, DTYPES))


def fields(n, is_pair=True, offsets=True, seq=True):
    """the first n FIELDS less type ids for single sequences, offsets where they are not returned and sequence ids where
    seq is False"""
    skip = {nm for nm, off in (("type_ids", is_pair), ("offsets", offsets), ("sequence_ids", seq)) if not off}
    return tuple(nm for nm in FIELDS[:n] if nm not in skip)


def kinds(x):
    """the truncation failures an error message names: PANIC (the stride check) and / or TOO_SHORT (SequenceTooShort)"""
    return {k for k in (PANIC, TOO_SHORT) if isinstance(x, str) and k in x}


def same(got, exp, what, names, ref=None):
    """rows (tuples in FIELDS order) or an error message, both sides; the fields in `names` are compared where got has them.
    ref: the restatement's result on the same batch (default exp), whose error message names every failure the batch's
    inputs hit.  The class of a truncation failure must match exactly, except on a batch that holds both a
    SequenceTooShort input and a stride panic: that may report either (the reference encodes the inputs in parallel,
    which one fails first is not defined).  A row that does not fit L is an error of its own class."""
    if isinstance(exp, str) or isinstance(got, str):
        ref = exp if ref is None else ref
        kg, ke, kr = kinds(got), kinds(exp), kinds(ref)
        trunc_ok = bool(kg) and bool(ke) and kg <= kr and ke <= kr and (len(kr) > 1 or kg == ke)
        fit_ok = isinstance(exp, str) and isinstance(got, str) and "fit" in exp and "fit" in got and not kg and not ke
        assert trunc_ok or fit_ok, (what, got if isinstance(got, str) else "rows", exp if isinstance(exp, str) else "rows", sorted(kr))
        return
    for nm, g, e in zip(FIELDS, got, exp):
        if nm in names and g is not None:
            assert g.shape == e.shape and np.array_equal(g, e), (what, nm, g.shape, e.shape)


def kept_rows(rows):
    """the rows of a result with overflowing parts that are each input's kept row"""
    kept = np.r_[True, np.diff(rows[4].astype(np.int64)) != 0] if len(rows[4]) else np.zeros(0, bool)
    return tuple(x[kept] for x in rows)


# ----------------------------------------------------------------------------------------- the kernels on the host
def emul():
    """native/dense_emul.cpp, built when it is older than its source or dense_kernels.cuh"""
    so = os.path.join(HERE, "native", "libdense_emul.so")
    src = os.path.join(HERE, "native", "dense_emul.cpp")
    hdr = os.path.join(helpers.ROOT, "tokenizers_b200", "csrc", "dense_kernels.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        inc = "/usr/local/cuda/include"
        if not os.path.exists(os.path.join(inc, "cuda_runtime.h")):
            pytest.skip("CUDA headers not available")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + inc, "-Wno-attributes", "-shared", "-fPIC", "-o", so, src])
    L = ctypes.CDLL(so)
    u32, vp, i32 = ctypes.c_uint32, ctypes.c_void_p, ctypes.c_int
    L.b2t_emul_pair_keep.restype = None; L.b2t_emul_pair_keep.argtypes = [u32] + [vp] * 7
    L.b2t_emul_seq_parts.restype = u32; L.b2t_emul_seq_parts.argtypes = [u32, u32, u32]
    L.b2t_emul_seq_part.restype = None; L.b2t_emul_seq_part.argtypes = [u32, u32, u32, i32, u32, vp, vp]
    L.b2t_emul_pair_row_part.restype = None; L.b2t_emul_pair_row_part.argtypes = [u32, u32, u32, vp, vp]
    L.b2t_emul_trim_span.restype = None; L.b2t_emul_trim_span.argtypes = [u32, u32, u32, u32, i32, i32, vp]
    L.b2t_emul_added_trim_counts.restype = i32; L.b2t_emul_added_trim_counts.argtypes = [u32] * 5 + [vp, vp]
    L.b2t_emul_dense_count.restype = ctypes.c_uint64; L.b2t_emul_dense_count.argtypes = [vp] + [u32] * 7 + [vp] * 4
    L.b2t_emul_dense_rows.restype = u32
    L.b2t_emul_dense_rows.argtypes = [vp] * 4 + [u32] * 5 + [vp] + [u32] * 5 + [i32, i32] + [u32] * 5 + [vp] + [u32] * 5 + [vp, vp, u32, u32] + [vp] * 9
    return L


# the emulated templates: special token ids above every sequence token, piece type ids (3, 4) other than the types of
# overflowing parts (0 for A, 1 for B)
EMUL_TEMPLATES = {
    "a_first": [("special", 900, 0), ("seq", 0, 3), ("special", 901, 0), ("seq", 1, 4), ("special", 902, 1)],
    "b_first": [("special", 900, 2), ("seq", 1, 4), ("special", 901, 0), ("special", 903, 0), ("seq", 0, 3), ("special", 900, 2)],
}

NS = (0, 1, 2, 5, 13, 40)   # sequence lengths of the emulated batches: pairs of every two of them


def single_template(pieces, n):
    """the first n pieces of the single-sequence template within an emulated pair template: its special tokens and A"""
    return [p for p in pieces if p[0] == "special" or p[1] == 0][:n]


def plain_batch(lens):
    """a CSR of documents with `lens` tokens (token t of document d = 1000 d + t, its offsets (t, t + 1)) in the layout of
    emul_rows: (ids, offsets, words, row_ptr, trim_vocab, trim_added, ld, tr), the token arrays with one entry past the end"""
    rp = np.zeros(len(lens) + 1, dtype=np.uint64); np.cumsum(lens, out=rp[1:])
    ids = np.concatenate([1000 * d + np.arange(n, dtype=np.uint32) for d, n in enumerate(lens)] + [np.zeros(1, np.uint32)]).astype(np.uint32)
    offs = np.concatenate([np.stack([np.arange(n), np.arange(n) + 1], axis=1) for n in lens] + [np.zeros((1, 2))]).astype(np.uint32)
    return ids, offs, None, rp, None, None, None, None


def emul_rows(L, batch, is_pair, pieces, budget, strategy, stride, left, *, over=True, offs=True, meta=False, aps=False, overflow_types=(0, 1),
              pad_left=False, width=None, err=0):
    """the length pass and the rows of the instance <over, offs, meta> on a batch (plain_batch's layout), padded to the
    width the length pass finds (or `width`) -> the nine FIELDS (None where the instance writes none) or the error
    message of the length pass.  err: the error bits the row kernels must raise."""
    ids, offsets, words, rp, tv, tab, _, _ = batch
    n_in = (len(rp) - 1) // (2 if is_pair else 1)
    n_sp = sum(1 for p in pieces if p[0] == "special")
    cnt = np.zeros(n_in + 1, dtype=np.uint32)
    mx, e, sm = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
    R = L.b2t_emul_dense_count(rp.ctypes.data, n_in, int(is_pair), int(over), budget, strategy, stride, n_sp, cnt.ctypes.data, ctypes.byref(mx),
                               ctypes.byref(e), ctypes.byref(sm))
    if e.value & 32:
        return TOO_SHORT
    if e.value & 64:
        return f"`stride` must be strictly less than `max_len={sm.value}`"
    W = mx.value if width is None else width
    seg, sp, b_first, tx, ty = [[], [], []], 0, 0, 0, 0
    for kind, v, t in pieces:
        if kind == "seq":
            if sp == 0:
                b_first, tx = int(v == 1), t
            else:
                ty = t
            sp += 1
        else:
            seg[sp].append(v | t << 24 if is_pair else v)
    if not is_pair:
        seg = [seg[0], [], seg[1]]   # pre A post
    special = np.asarray(seg[0] + seg[1] + seg[2] + [0], dtype=np.uint32)
    out = np.zeros((R, W), np.uint32); tout = np.zeros((R, W), np.uint8); mask = np.zeros((R, W), np.uint8)
    olen = np.zeros(R + 1, np.uint32); samp = np.zeros(R + 1, np.uint32); ooff = np.zeros((R, W, 2), np.uint32)
    osp = np.zeros((R, W), np.uint8); oseq = np.zeros((R, W), np.int8); owd = np.zeros((R, W), np.uint32)
    ptr = lambda a: None if a is None else a.ctypes.data
    got = L.b2t_emul_dense_rows(ids.ctypes.data, offsets.ctypes.data, ptr(words), rp.ctypes.data, n_in, int(is_pair), int(over), int(offs), int(meta),
                                cnt.ctypes.data, R, W, budget, strategy, stride, int(left), int(pad_left), 7, 5, len(seg[0]), len(seg[1]), len(seg[2]),
                                special.ctypes.data, b_first, tx, ty, overflow_types[0], overflow_types[1], ptr(tv), ptr(tab), 0 if tab is None else len(tab),
                                int(aps), out.ctypes.data, tout.ctypes.data, mask.ctypes.data, olen.ctypes.data, samp.ctypes.data, ooff.ctypes.data,
                                osp.ctypes.data, oseq.ctypes.data, owd.ctypes.data)
    assert got == err, (got, err)
    return (out, tout if is_pair else None, mask, olen[:R], samp[:R] if over else None, ooff if offs else None, osp if meta else None,
            oseq if meta else None, owd.view(np.int32) if meta else None)


def restated_rows(batch, is_pair, pieces, budget, strategy, stride, left, *, over=True, trim=None, overflow_type=None, pad_left=False):
    """the same batch through dense_oracle.dense_meta_rows (pairs.post_process), the added-token marks cleared, padded to
    the longest row of all (over), or the kept rows alone padded to the longest of them.  trim: the template's
    add_prefix_space rule for offset trimming, None = no trimming; overflow_type: the type id a RobertaProcessing-style
    template gives every overflowing part"""
    ids, offs, words, rp, _, _, ld, tr = batch
    single = None if is_pair else pieces
    tpl = {"pair": pieces, "single": single, "trim": trim, "pre": [], "post": [], "overflow_type": overflow_type}
    trn = dict(max_length=budget + sum(1 for p in (pieces if is_pair else single) if p[0] == "special"), stride=stride, strategy=strategy,
               direction="left" if left else "right")
    out = dense_oracle.dense_meta_rows(ids[:-1] & np.uint32(0x7FFFFFFF), offs[:-1], None if words is None else words[:-1], rp, ld, tr,
                                       is_pair=is_pair, template=tpl, truncation=trn, add_special_tokens=True, pad_all_rows=True,
                                       padding=dict(length=None, direction="left" if pad_left else "right", pad_id=7, pad_type_id=5))
    if isinstance(out, str) or over:
        return out
    out = kept_rows(out)
    w = int(out[3].max(initial=0))
    cols = slice(out[0].shape[1] - w, None) if pad_left else slice(0, w)   # (an overflowing part may be longer than any kept row)
    return tuple(x[:, cols] if x.ndim > 1 else x for x in out)
