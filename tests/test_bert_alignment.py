"""BertNormalizer's per-character alignment -- the original character behind every normalized character, which N3 maps token
offsets back through -- against the reference wheel.  Token offsets only show the alignment of a token's first and last
character; these tests compare every character.

The reference: a WordLevel model with only [UNK] behind the variant's BertNormalizer and a pre-tokenizer that isolates every
character, so that each token is one normalized character and its offsets are that character's original range.

- CPU: the oracle's restatement (text and alignment) on every scalar value and on every run of combining marks NFD can
  reorder; the kernels' own N1 refusal and N3 mapping through a host emulator (tests/native/norm_emul.cpp): where N1 accepts
  a run, the kernels' model -- the image table, every output character aligned with its own input character -- must be the
  reference's.
- GPU: the bert pipeline (BertPreTokenizer + WordPiece) against the wheel on ids, offsets, word ids and row_ptr for every
  scalar value, all accepted runs, refused runs and survivors placed across thread chunks, pages and documents."""
import ctypes, functools, os, random, subprocess, unicodedata
import numpy as np
import pytest
import helpers
from oracle import oracle as orc

tk = helpers.wheel()
HERE = os.path.dirname(os.path.abspath(__file__))

VARIANTS = {"uncased": dict(clean_text=True, handle_chinese_chars=True, strip_accents=None, lowercase=True),
            "cased": dict(clean_text=True, handle_chinese_chars=True, strip_accents=False, lowercase=False),
            "strip_only": dict(clean_text=False, handle_chinese_chars=False, strip_accents=True, lowercase=False),
            "clean_strip": dict(clean_text=True, handle_chinese_chars=False, strip_accents=True, lowercase=False)}
STRIP = ["uncased", "strip_only", "clean_strip"]
needs_wheel = pytest.mark.skipif(tk is None, reason="reference wheel not importable")

# runs the parent's oracle and N1 got wrong (a survivor -- a mark strip_accents keeps -- that canonical ordering moves, or
# that moves another mark), with the character the reference aligns the survivor with
TABLE = [("a\u08d4\u0316x", 2), ("a\u08d4\x01\u0316x", 3), ("a\u0301\x01\u302ex", 1), ("a\u08d4\u0f73x", 2),
         ("a\u0345\u08d4x", 1), ("x\u0301\u302ey", 1), ("a\u0316\u08d4x", 2)]


def _flags_bits(flags):
    nz = orc.BertNormalizer(**flags)
    return (1 if nz.clean else 0) | (2 if nz.chinese else 0) | (4 if nz.strip else 0) | (8 if nz.lower else 0)


@functools.lru_cache(maxsize=None)
def _aligner(variant):
    t = tk.Tokenizer(tk.models.WordLevel({"[UNK]": 0}, unk_token="[UNK]"))
    t.normalizer = tk.normalizers.BertNormalizer(**VARIANTS[variant])
    t.pre_tokenizer = tk.pre_tokenizers.Split(tk.Regex("[\\s\\S]"), "isolated")   # (Oniguruma rejects (?s).)
    return t


def wheel_alignment(variant, docs):
    """the wheel over docs laid end to end: normalized text, and the original character range [start, end) of each of its
    characters, counted from the start of the first document"""
    t = _aligner(variant)
    encs = t.encode_batch(docs, add_special_tokens=False)
    base, al = 0, []
    for d, e in zip(docs, encs):
        al += [(a + base, b + base) for a, b in e.offsets]
        base += len(d)
    return "".join(t.normalizer.normalize_str(d) for d in docs), np.array(al, dtype=np.int64).reshape(-1, 2)


def _char_index(raw):
    """byte offset -> number of characters that start in front of it (len(raw) + 1 entries)"""
    r = np.frombuffer(raw, dtype=np.uint8)
    return np.concatenate([[0], np.cumsum((r & 0xC0) != 0x80)])


def oracle_alignment(variant, docs):
    """oracle.BertNormalizer.normalize in the same form (the documents are normalized one after the other)"""
    nz = orc.BertNormalizer(**VARIANTS[variant])
    texts, als, base = [], [], 0
    for d in docs:
        raw = d.encode("utf-8")
        out, al = nz.normalize(raw)
        o = np.frombuffer(out, dtype=np.uint8)
        texts.append(out.decode("utf-8"))
        als.append(_char_index(raw)[al[(o & 0xC0) != 0x80].astype(np.int64)] + base)
        base += len(d)
    return "".join(texts), (np.concatenate(als) if als else np.zeros((0, 2), np.int64)).reshape(-1, 2)


@functools.lru_cache(maxsize=None)
def images(variant):
    """the image of every code point as the kernels' table holds it (b2t_bert_normalizer_images: host only)"""
    from tokenizers_b200 import _lib
    pool = np.zeros(6 << 20, dtype=np.uint8); off = np.zeros(0x110001, dtype=np.uint32)
    _lib.check(_lib.lib().b2t_bert_normalizer_images(_flags_bits(VARIANTS[variant]), pool.ctypes.data, pool.size, off.ctypes.data))
    return pool.tobytes(), off


def model_alignment(variant, docs):
    """what the kernels compute where N1 accepts: the image of every character, each output character aligned with its own
    input character"""
    raw, off = images(variant)
    text, al, base = [], [], 0
    for d in docs:
        for k, ch in enumerate(d):
            c = ord(ch)
            im = raw[off[c]:off[c + 1]].decode("utf-8")
            text.append(im)
            al += [(base + k, base + k + 1)] * len(im)
        base += len(d)
    return "".join(text), np.array(al, dtype=np.int64).reshape(-1, 2)


def _assert_same(exp, got, docs, what):
    (te, ae), (tg, ag) = exp, got
    if te == tg and np.array_equal(ae, ag):
        return
    starts = np.cumsum([0] + [len(d) for d in docs])
    n = min(len(te), len(tg))
    i = next((k for k in range(n) if te[k] != tg[k] or tuple(ae[k]) != tuple(ag[k])), n)
    src = ae[i][0] if i < len(ae) else ag[i][0]
    d = int(np.searchsorted(starts, src, side="right") - 1)
    raise AssertionError(f"{what}: normalized character {i} differs: reference {te[i:i + 1]!r} {ae[i:i + 1].tolist()} "
                         f"got {tg[i:i + 1]!r} {ag[i:i + 1].tolist()}; document {d} {[hex(ord(c)) for c in docs[d]]}")


def every_scalar():
    return [c for c in range(0x110000) if not 0xD800 <= c <= 0xDFFF]


def survivors():
    nz = orc.BertNormalizer(**VARIANTS["uncased"])
    s = [c for c in every_scalar() if nz._ccc[c] and not nz._mn[c]]
    assert len(s) == 83
    return s


@functools.lru_cache(maxsize=None)
def mark_runs():
    """every run of marks in which canonical ordering can move a survivor (S) or move another mark past it.  X: every code
    point whose NFD holds a non-zero class (Python's unicodedata; the wheel decides what happens), S and U+0345.
    S X and X S adjacent and with a character clean_text removes between them; a seeded sample of three-mark runs; a
    precomposed character with trailing marks in front of S.  Each run sits between two base characters."""
    S = survivors()
    X = sorted(set(c for c in every_scalar() if any(unicodedata.combining(ch) for ch in unicodedata.normalize("NFD", chr(c))))
               | set(S) | {0x345})
    runs = [r for r, _ in TABLE]
    for s in map(chr, S):
        for x in map(chr, X):
            for sep in ("", "\x01", "\x00", "\ufffd"):
                runs += ["a" + s + sep + x + "b", "a" + x + sep + s + "b"]
    rng = random.Random(11)
    pool = [chr(c) for c in X]
    for _ in range(30000):
        m = [rng.choice(pool) for _ in range(3)]
        m[rng.randrange(3)] = chr(rng.choice(S))
        runs.append("x" + "".join(m) + "y")
    pre = [chr(c) for c in every_scalar() if len(unicodedata.normalize("NFD", chr(c))) >= 3
           and unicodedata.combining(unicodedata.normalize("NFD", chr(c))[0]) == 0]
    for p in pre:
        for s in map(chr, S[::7]):
            runs += [p + s + "z", "z" + p + s]
    runs += ["\u1ec7" + chr(s) + "z" for s in S]
    return runs


def _pack(runs, per_doc=256):
    return [" ".join(runs[i:i + per_doc]) for i in range(0, len(runs), per_doc)]


# ------------------------------------------------------------------------------------------------------- the oracle
@needs_wheel
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("run,char", TABLE)
def test_oracle_table_cases(variant, run, char):
    exp = wheel_alignment(variant, [run])
    _assert_same(exp, oracle_alignment(variant, [run]), [run], f"oracle vs wheel, {variant}")
    if variant in ("uncased", "clean_strip"):   # (the rows with U+0001 need clean_text)
        s = next(k for k, ch in enumerate(run) if ord(ch) in (0x8D4, 0x302E))
        assert [tuple(a) for t, a in zip(exp[0], exp[1]) if t == run[s]] == [(char, char + 1)]


@needs_wheel
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_oracle_alignment_every_scalar_value(variant):
    """all 1 112 064 scalar values, each as "x" + c + " ": normalized text and the alignment of every character"""
    docs = ["x" + chr(c) + " " for c in every_scalar()]
    exp = wheel_alignment(variant, docs)
    big = ["".join(docs[i:i + 4096]) for i in range(0, len(docs), 4096)]   # (the pieces are independent: the oracle runs on fewer, longer strings)
    _assert_same(exp, oracle_alignment(variant, big), docs, f"oracle vs wheel, every scalar value, {variant}")


@needs_wheel
@pytest.mark.parametrize("variant", STRIP)
def test_oracle_alignment_mark_runs(variant):
    docs = _pack(mark_runs())
    _assert_same(wheel_alignment(variant, docs), oracle_alignment(variant, docs), docs, f"oracle vs wheel, mark runs, {variant}")


# ------------------------------------------------------------------------------------------- the kernels, emulated
@functools.lru_cache(maxsize=None)
def _emul():
    so = os.path.join(HERE, "native", "libnorm_emul.so")
    srcs = [os.path.join(HERE, "native", "norm_emul.cpp")] + [os.path.join(helpers.ROOT, "tokenizers_b200", "csrc", f)
                                                              for f in ("norm_kernels.cuh", "b2t_tables.h", "host_tables.cu", "bert_tables.inc")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(map(os.path.getmtime, srcs)):
        inc = "/usr/local/cuda/include"
        if not os.path.exists(os.path.join(inc, "cuda_runtime.h")):
            pytest.skip("CUDA headers not available")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + inc, "-Wno-attributes", "-shared", "-fPIC", "-include", "cuda_runtime.h",
                               "-o", so, srcs[0], "-x", "c++", srcs[3]])
    L = ctypes.CDLL(so)
    vp = ctypes.c_void_p
    L.b2t_emul_norm_tables.restype = ctypes.c_int; L.b2t_emul_norm_tables.argtypes = [ctypes.c_int]
    L.b2t_emul_norm_refused.restype = None; L.b2t_emul_norm_refused.argtypes = [vp, vp, ctypes.c_uint32, vp, vp, vp]
    L.b2t_emul_norm_offsets.restype = None; L.b2t_emul_norm_offsets.argtypes = [vp, ctypes.c_uint32, vp, vp, vp, vp]
    return L


def emul_refused(variant, batches):
    """N1's refusal bit of every batch (a list of strings, each its own batch), and N1's image byte count of each"""
    L = _emul()
    assert L.b2t_emul_norm_tables(_flags_bits(VARIANTS[variant])) == 0
    data, off = helpers.pack_docs(batches)
    data = np.concatenate([data, np.zeros(16, np.uint8)])
    ref, n_out, n_chars = np.zeros(len(batches), np.uint8), np.zeros(len(batches), np.uint64), np.zeros(len(batches), np.uint64)
    L.b2t_emul_norm_refused(data.ctypes.data, off.ctypes.data, len(batches), ref.ctypes.data, n_out.ctypes.data, n_chars.ctypes.data)
    assert np.array_equal(n_chars, [len(b) for b in batches])
    return ref.astype(bool), n_out


def run_outcome(variant, runs):
    """per run: refused by N1 alone, and whether the kernels' model differs from the wheel"""
    refused, n_out = emul_refused(variant, runs)
    te, ae = wheel_alignment(variant, runs)
    tm, am = model_alignment(variant, runs)
    _, off = images(variant)
    assert len(te) == len(tm) and np.array_equal(n_out, [sum(int(off[ord(c) + 1] - off[ord(c)]) for c in r) for r in runs])
    starts = np.cumsum([0] + [len(r) for r in runs])
    bad = np.zeros(len(runs), bool)
    diff = np.nonzero((np.frombuffer(te.encode("utf-32-le"), np.uint32) != np.frombuffer(tm.encode("utf-32-le"), np.uint32)) | (ae != am).any(axis=1))[0]
    for a in (ae, am):
        bad[np.searchsorted(starts, a[diff, 0], side="right") - 1] = True
    return refused, bad


@needs_wheel
@pytest.mark.parametrize("variant", STRIP)
def test_kernels_refuse_every_run_they_would_align_differently(variant):
    """every mark run as its own batch: where N1 accepts, the image table with each character aligned to itself is what the
    reference computes"""
    runs = mark_runs()
    refused, bad = run_outcome(variant, runs)
    wrong = [runs[i] for i in np.nonzero(bad & ~refused)[0]]
    assert not wrong, [[hex(ord(c)) for c in r] for r in wrong[:5]]
    for r, _ in TABLE:   # (without clean_text, U+0001 is a character of its own between the marks)
        assert refused[runs.index(r)] or not VARIANTS[variant]["clean_text"], [hex(ord(c)) for c in r]
    print(f"{variant}: {int(refused.sum())} of {len(runs)} runs refused, {int(bad.sum())} would be aligned differently")


@needs_wheel
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_kernels_every_scalar_value(variant):
    """every scalar value in context: N1 never refuses a batch without a survivor, accepts a survivor between base characters,
    and the model is the reference's"""
    docs = ["x" + chr(c) + " " for c in every_scalar()]
    refused, _ = emul_refused(variant, docs)
    assert not refused.any(), [hex(ord(docs[i][1])) for i in np.nonzero(refused)[0][:10]]
    big = ["".join(docs[i:i + 4096]) for i in range(0, len(docs), 4096)]
    assert not emul_refused(variant, big)[0].any()
    _assert_same(wheel_alignment(variant, docs), model_alignment(variant, big), docs, f"kernel model vs wheel, {variant}")


@needs_wheel
@pytest.mark.parametrize("variant", STRIP)
def test_norm_offsets_kernel_maps_every_character(variant):
    """N3 on tokens of one normalized character each, src_char / doc_char0 as N2 writes them for accepted runs: the
    character offsets are the reference's"""
    runs = mark_runs()[::53]
    refused, _ = emul_refused(variant, runs)
    docs = [r for r, x in zip(runs, refused) if not x]
    te, ae = wheel_alignment(variant, docs)
    raw, off = images(variant)
    src, doc_off_norm, doc_char0, row_ptr, offs = [], [0], [0], [0], []
    gchar = 0
    for d in docs:
        pos = 0
        for ch in d:
            im = raw[off[ord(ch)]:off[ord(ch) + 1]]
            src += [gchar] * len(im)
            for k in range(len(im)):
                if (im[k] & 0xC0) != 0x80:
                    l = 1 + sum(1 for b in im[k + 1:k + 4] if (b & 0xC0) == 0x80) if im[k] >= 0x80 else 1
                    offs.append((pos + k, pos + k + l))
            pos += len(im); gchar += 1
        doc_off_norm.append(doc_off_norm[-1] + pos); doc_char0.append(gchar); row_ptr.append(len(offs))
    src = np.array(src + [0], np.uint32); offs = np.array(offs, np.uint32).reshape(-1, 2).copy()
    dn, dc, rp = np.array(doc_off_norm, np.uint64), np.array(doc_char0, np.uint32), np.array(row_ptr, np.uint64)
    _emul().b2t_emul_norm_offsets(rp.ctypes.data, len(docs), dn.ctypes.data, dc.ctypes.data, src.ctypes.data, offs.ctypes.data)
    starts = np.repeat(np.cumsum([0] + [len(d) for d in docs])[:-1], np.diff(rp).astype(np.int64))
    assert np.array_equal(offs.astype(np.int64) + starts[:, None], ae)


# ----------------------------------------------------------------------------------------------------------- GPU
def _wheel_bert(variant):
    return tk.Tokenizer.from_str(helpers.bert_json(VARIANTS[variant]))


def _gpu_tok(variant):
    from tokenizers_b200 import Tokenizer
    return Tokenizer.from_str(helpers.bert_json(VARIANTS[variant]))


def _gpu_vs_wheel(tok, wt, docs, what):
    be = tok.encode_batch_csr(*helpers.pack_docs(docs))
    helpers.assert_csr_equal((be.ids, be.offsets, be.word_ids, be.row_ptr), helpers.wheel_csr(wt, docs), docs, what)


def _refused_on_gpu(tok, docs):
    from tokenizers_b200 import _lib
    try:
        tok.encode_batch_csr(*helpers.pack_docs(docs))
    except _lib.B2TError as ex:
        assert ex.code == _lib.B2T_ERR_UNSUPPORTED and "combining character" in str(ex), str(ex)
        return True
    return False


@pytest.mark.gpu
@needs_wheel
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_gpu_every_scalar_value(variant):
    tok, wt = _gpu_tok(variant), _wheel_bert(variant)
    for form in (lambda c: "x" + c + " ", lambda c: c + "x "):
        _gpu_vs_wheel(tok, wt, [form(chr(c)) for c in every_scalar()], f"every scalar value, {variant}")


@pytest.mark.gpu
@needs_wheel
@pytest.mark.parametrize("variant", STRIP)
def test_gpu_mark_runs(variant):
    """all runs N1 accepts in one batch (one run per document) against the wheel; a few of each kind it refuses, each in a
    small batch of its own, refused on the device"""
    from tokenizers_b200 import _lib
    runs = mark_runs()
    refused, bad = run_outcome(variant, runs)
    tok, wt = _gpu_tok(variant), _wheel_bert(variant)
    _gpu_vs_wheel(tok, wt, [r for r, x in zip(runs, refused) if not x], f"accepted mark runs, {variant}")
    rng = random.Random(3)
    kinds = {}
    for i in np.nonzero(refused)[0]:
        kinds.setdefault((bool(bad[i]), len(runs[i]), runs[i][2] if len(runs[i]) > 3 else ""), []).append(runs[i])
    picks = [r for r, _ in TABLE if refused[runs.index(r)]] + [r for v in kinds.values() for r in rng.sample(v, min(2, len(v)))]
    for r in picks[:400]:
        assert _refused_on_gpu(tok, ["fine", r, "also fine"]), [hex(ord(c)) for c in r]


@pytest.mark.gpu
@needs_wheel
@pytest.mark.parametrize("variant", ["uncased", "clean_strip"])
def test_gpu_survivor_edges(variant):
    """a survivor and its neighbour across an 8-byte thread chunk, a 2 KB page and a document boundary, and as the last
    character of the batch: correct or refused, never wrong; with base characters around it, accepted"""
    tok, wt = _gpu_tok(variant), _wheel_bert(variant)
    accept = ["a\u08d4b", "a\u302e", "\u08d4z", "\u1ec7\u08d4q", "\u0915\u08e1 \u08e0"]
    mixed = ["\u0316\u08d4", "\u08d4\u0316", "\u08d4\x01", "\x01\u302e", "\u08d4\u08d5", "\u0345\u08d4"]
    for probe in accept + mixed:
        for form in ("doc", "text"):
            for delta in range(-7, 8):
                for anchor in ("start", "end"):
                    docs = helpers.place([(probe, helpers.PAGE + delta, anchor), ("x" + probe + "y", 2 * helpers.PAGE + 8 + delta, "end")], form)
                    if probe in accept and form == "text":
                        _gpu_vs_wheel(tok, wt, docs, f"{probe!r} at {delta} {anchor} {variant}")
                    elif not _refused_on_gpu(tok, docs):
                        _gpu_vs_wheel(tok, wt, docs, f"{probe!r} at {delta} {anchor} ({form}) {variant}")
    # across a document boundary, and the batch's last character
    for docs in (["x\u0316", "\u08d4x"], ["x\u08d4", "\u0316x"], ["x\x01", "\u08d4"], ["ab", "\u08d4"], ["x\u08d4"], ["\u08d4"],
                 ["y" * 2046 + "\u08d4"], ["y" * 2047 + "\u08d4"], ["y" * 2045, "\u08d4"], ["q\u08d4", "\u08d4q"]):
        if not _refused_on_gpu(tok, docs):
            _gpu_vs_wheel(tok, wt, docs, f"{docs!r} {variant}")
    assert not _refused_on_gpu(tok, ["ab", "\u08d4"]) and not _refused_on_gpu(tok, ["y" * 2047 + "\u08d4"])
