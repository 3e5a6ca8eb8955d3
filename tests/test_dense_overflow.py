"""Dense mode with overflowing parts and offset rows (B2T_DENSE_OVERFLOW, B2T_DENSE_OFFSETS): stride truncation of single
sequences and pairs, the rows of every part in the reference's order, the sample map and the char offsets of every position.
CPU: the part algebra and the row kernels of dense_kernels.cuh (run on the host by tests/native/overflow_emul.cpp) against
the shim's host restatement (truncation_spans, pairs.post_process); the restatement tests/overflow_oracle.py against the
reference wheel and the committed fixture; the spec the shim builds.  GPU: the engine against all of them."""
import ctypes, gzip, json, os, random, subprocess
import numpy as np
import pytest
import helpers, corpus
import test_dense_pairs as tdp
import overflow_oracle as oo
from oracle import oracle as orc
from tokenizers_b200 import pairs as shim_pairs
from tokenizers_b200.tokenizer import parse_post_processor, special_token_count, truncation_spans

tk = helpers.wheel()
HERE = os.path.dirname(os.path.abspath(__file__))
STRATEGIES = tdp.STRATEGIES
PANIC = "must be strictly less than `max_len"
TOO_SHORT = "too short to respect"
NOT_FIT = "does not fit"

# (truncation, padding).  stride "b-1": the budget (max_length less the template's special tokens) - 1, where every cut
# sequence panics under only_first / only_second (its max_len is below the budget) and longest_first panics on some pairs.
SETTINGS = [
    (dict(max_length=24, stride=0, strategy="longest_first", direction="right"), dict(length=24, direction="right", pad_id=0, pad_type_id=0)),
    (dict(max_length=20, stride=1, strategy="only_second", direction="left"), dict(length=None, direction="left", pad_id=3, pad_type_id=1, pad_to_multiple_of=8)),
    (dict(max_length=28, stride=5, strategy="only_first", direction="right"), dict(length=None, direction="right", pad_id=1, pad_type_id=2)),
    (dict(max_length=30, stride=4, strategy="longest_first", direction="left"), dict(length=32, direction="right", pad_id=2, pad_type_id=0)),
    (dict(max_length=26, stride="b-1", strategy="only_second", direction="right"), dict(length=None, direction="right", pad_id=2, pad_type_id=0)),
    (dict(max_length=26, stride="b-1", strategy="longest_first", direction="right"), dict(length=None, direction="right", pad_id=2, pad_type_id=0)),
]


def resolve(js, tr, is_pair, ast):
    """the setting with its stride resolved against the template's budget (the reference's enable_truncation refuses a
    stride that is not below max_length less the special tokens of a single sequence)"""
    if tr["stride"] != "b-1":
        return tr
    tp = parse_post_processor(json.loads(js).get("post_processor"))
    budget = tr["max_length"] - (special_token_count(tp, is_pair) if ast else 0)
    return dict(tr, stride=max(min(budget, tr["max_length"] - special_token_count(tp, False)) - 1, 0))


def arrange(seqs, tr, is_pair):
    return tdp.arrange(seqs, tr) if is_pair else [a for a, _ in seqs]


def cases():
    for k, (tr, pd) in enumerate(SETTINGS):
        for is_pair in (True, False):
            if not is_pair and tr["strategy"] == "only_second":
                continue   # (a single sequence has no second one to cut: the reference refuses)
            for ast in (True, False):
                yield f"{k}/{'pair' if is_pair else 'single'}/{int(ast)}", tr, pd, is_pair, ast


def inputs_for(seed, n=60):
    """pairs of a fuzz document and a short sentence, long contexts that make many windows, and the empty corner cases"""
    ps = tdp.pairs_for(seed, n)
    rng = random.Random(seed)
    long_ = [" ".join(rng.choice(tdp.WORDS) for _ in range(rng.randint(40, 120))) for _ in range(4)]
    return ps + [(t, "why not") for t in long_]


def flat(x):
    return [s for p in x for s in (p if isinstance(p, (tuple, list)) else (p,))]


def oracle_rows(js, inputs, tr, pd, is_pair, ast):
    ids, offs, _, rp = orc.Oracle(js).encode_batch(flat(inputs))
    tp = parse_post_processor(json.loads(js).get("post_processor"))
    return oo.dense_overflow_rows(ids, offs, rp, is_pair=is_pair, template=tp, truncation=tr, padding=pd, add_special_tokens=ast)


def wheel_rows(js, inputs, tr, pd, ast):
    """the reference: encode_batch with truncation (stride) and padding, every input's Encoding and its overflowing
    Encodings stacked in that order"""
    tok = tk.Tokenizer.from_str(js)
    tok.enable_truncation(tr["max_length"], stride=tr["stride"], strategy=tr["strategy"], direction=tr["direction"])
    tok.enable_padding(direction=pd["direction"], pad_id=pd["pad_id"], pad_type_id=pd["pad_type_id"], length=pd["length"],
                       pad_to_multiple_of=pd.get("pad_to_multiple_of"))
    try:
        encs = tok.encode_batch(inputs, add_special_tokens=ast)
    except BaseException as ex:   # (the stride check is a Rust panic: PanicException derives from BaseException)
        if isinstance(ex, (KeyboardInterrupt, SystemExit)):
            raise
        return str(ex)
    rows, sample = [], []
    for p, e in enumerate(encs):
        for x in [e] + list(e.overflowing):
            rows.append(x); sample.append(p)
    widths = {len(x.ids) for x in rows}
    if len(widths) > 1:
        return f"rows of {sorted(widths)} tokens: a row does not fit L"
    R, L = len(rows), widths.pop() if widths else 0
    return (np.array([x.ids for x in rows], dtype=np.uint32).reshape(R, L), np.array([x.type_ids for x in rows], dtype=np.uint8).reshape(R, L),
            np.array([x.attention_mask for x in rows], dtype=np.uint8).reshape(R, L), np.array([sum(x.attention_mask) for x in rows], dtype=np.uint32),
            np.array(sample, dtype=np.uint32), np.array([x.offsets for x in rows], dtype=np.uint32).reshape(R, L, 2))


FIELDS = ("ids", "type_ids", "mask", "lengths", "sample", "offsets")


def kinds(x):
    """the truncation failures an error message names: PANIC (the stride check) and / or TOO_SHORT (SequenceTooShort)"""
    return {k for k in (PANIC, TOO_SHORT) if isinstance(x, str) and k in x}


def same(got, exp, what, is_pair=True, offsets=True, ref=None):
    """(ids, type ids, mask, lengths, sample, offsets) or an error message, both sides; type ids / offsets are compared
    where the engine returns them.  ref: the restatement's result on the same batch (default exp), whose error message
    names every failure the batch's inputs hit.  The class of a truncation failure must match exactly, except on a batch
    that holds both a SequenceTooShort input and a stride panic: that may report either (the reference encodes the inputs
    in parallel, which one fails first is not defined)."""
    if isinstance(exp, str) or isinstance(got, str):
        ref = exp if ref is None else ref
        kg, ke, kr = kinds(got), kinds(exp), kinds(ref)
        trunc_ok = bool(kg) and bool(ke) and kg <= kr and ke <= kr and (len(kr) > 1 or kg == ke)
        fit_ok = isinstance(exp, str) and isinstance(got, str) and "fit" in exp and "fit" in got and not kg and not ke
        assert trunc_ok or fit_ok, (what, got if isinstance(got, str) else "rows", exp if isinstance(exp, str) else "rows", sorted(kr))
        return
    for g, e, nm in zip(got, exp, FIELDS):
        if g is None or (nm == "type_ids" and not is_pair) or (nm == "offsets" and not offsets):
            continue
        assert g.shape == e.shape and np.array_equal(g, e), (what, nm, g.shape, e.shape)


def _golden():
    return json.loads(gzip.open(os.path.join(helpers.GOLDEN, "golden_dense_overflow.json.gz")).read().decode("utf-8"))


def golden_rows(c):
    if "error" in c:
        return c["error"]
    R, L = c["shape"]
    return (np.array(c["ids"], dtype=np.uint32).reshape(R, L), np.array(c["type_ids"], dtype=np.uint8).reshape(R, L),
            np.array(c["mask"], dtype=np.uint8).reshape(R, L), np.array(c["lengths"], dtype=np.uint32), np.array(c["sample"], dtype=np.uint32),
            np.array(c["offsets"], dtype=np.uint32).reshape(R, L, 2))


def trimmed(name):
    """the templates whose post-processor trims offsets: offset rows are refused there"""
    tp = parse_post_processor(json.loads(tdp.tokenizer_json(name)).get("post_processor"))
    return tp is not None and tp["trim"] is not None


# ------------------------------------------------------------------------------------------------------------- CPU
def _emul():
    so = os.path.join(HERE, "native", "liboverflow_emul.so")
    src = os.path.join(HERE, "native", "overflow_emul.cpp")
    hdr = os.path.join(helpers.ROOT, "tokenizers_b200", "csrc", "dense_kernels.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        inc = "/usr/local/cuda/include"
        if not os.path.exists(os.path.join(inc, "cuda_runtime.h")):
            pytest.skip("CUDA headers not available")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + inc, "-Wno-attributes", "-shared", "-fPIC", "-o", so, src])
    L = ctypes.CDLL(so)
    u32, vp = ctypes.c_uint32, ctypes.c_void_p
    L.b2t_emul_seq_parts.restype = u32; L.b2t_emul_seq_parts.argtypes = [u32, u32, u32]
    L.b2t_emul_seq_part.restype = None; L.b2t_emul_seq_part.argtypes = [u32, u32, u32, ctypes.c_int, u32, vp, vp]
    L.b2t_emul_pair_row_part.restype = None; L.b2t_emul_pair_row_part.argtypes = [u32, u32, u32, vp, vp]
    L.b2t_emul_overflow_count.restype = ctypes.c_uint64
    L.b2t_emul_overflow_count.argtypes = [vp, u32, u32, u32, u32, u32, u32, vp, vp, vp, vp]
    L.b2t_emul_overflow_rows.restype = None
    L.b2t_emul_overflow_rows.argtypes = [vp, vp, vp, u32, u32, vp, u32, u32, u32, u32, u32, ctypes.c_int, ctypes.c_int, u32, u32, u32, u32, u32, vp,
                                         u32, u32, u32, u32, u32, u32, vp, vp, vp, vp, vp, vp]
    return L


def test_seq_part_algebra_exhaustive():
    """seq_parts / seq_part == truncation_spans (Encoding::truncate) for every n in [0, 40], max_len in [0, 48], stride in
    [0, 48] and both directions, the stride panic included"""
    L = _emul()
    f, ln = ctypes.c_uint32(), ctypes.c_uint32()
    for n in range(41):
        for m in range(49):
            for s in range(49):
                cnt = L.b2t_emul_seq_parts(n, m, s)
                for direction in ("right", "left"):
                    try:
                        exp = truncation_spans(n, m, s, direction)
                    except ValueError:
                        assert cnt == 0, (n, m, s)
                        continue
                    assert cnt == len(exp), (n, m, s, cnt, exp)
                    for k, (a, b) in enumerate(exp):
                        L.b2t_emul_seq_part(n, m, s, direction == "left", k, ctypes.byref(f), ctypes.byref(ln))
                        assert (f.value, f.value + ln.value) == (a, b), (n, m, s, direction, k)


def test_pair_row_order_matches_merge_with():
    """pair_row_part == the order of the rows pairs.merge_with (Encoding::merge_with) makes, for o_x, o_y in [0, 12]"""
    L = _emul()
    i, j = ctypes.c_uint32(), ctypes.c_uint32()

    def seq(label, o):
        e = shim_pairs.PE([(label, 0)], [0], [0], [(0, 0)], [0], [1], [0])
        e.overflowing = [shim_pairs.PE([(label, k)], [0], [0], [(0, 0)], [0], [1], [0]) for k in range(1, o + 1)]
        return e
    for ox in range(13):
        for oy in range(13):
            acc = shim_pairs.PE()
            shim_pairs.merge_with(acc, seq("x", ox))
            shim_pairs.merge_with(acc, seq("y", oy))
            exp = [(e.ids[0][1], e.ids[1][1]) for e in [acc] + acc.overflowing]
            assert len(exp) == (1 + ox) * (1 + oy)
            for r, ij in enumerate(exp):
                L.b2t_emul_pair_row_part(r, ox, oy, ctypes.byref(i), ctypes.byref(j))
                assert (i.value, j.value) == ij, (ox, oy, r)


# the emulated templates: special token ids above every sequence token, piece type ids (3, 4) other than the types of
# overflowing parts (0 for A, 1 for B)
EMUL_TEMPLATES = {
    "a_first": [("special", 900, 0), ("seq", 0, 3), ("special", 901, 0), ("seq", 1, 4), ("special", 902, 1)],
    "b_first": [("special", 900, 2), ("seq", 1, 4), ("special", 901, 0), ("special", 903, 0), ("seq", 0, 3), ("special", 900, 2)],
}


def emul_rows(L, lens, is_pair, pieces, budget, strategy, stride, left, overflow_types, pad_left=False):
    """the emulated kernels on a batch whose sequences have `lens` tokens (token t of document d = 1000 d + t, its offsets
    (t, t + 1)), padded to the longest row of all -> (ids, type ids, mask, lengths, sample, offsets) or an error tag"""
    per = 2 if is_pair else 1
    n_in = len(lens) // per
    rp = np.zeros(len(lens) + 1, dtype=np.uint64); np.cumsum(lens, out=rp[1:])
    ids = np.concatenate([1000 * d + np.arange(n, dtype=np.uint32) for d, n in enumerate(lens)] + [np.zeros(1, np.uint32)]).astype(np.uint32)
    offs = np.concatenate([np.stack([np.arange(n), np.arange(n) + 1], axis=1) for n in lens] + [np.zeros((1, 2))]).astype(np.uint32)
    n_special = sum(1 for p in pieces if p[0] == "special")
    cnt = np.zeros(n_in + 1, dtype=np.uint32)
    mx, err, sm = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
    R = L.b2t_emul_overflow_count(rp.ctypes.data, n_in, int(is_pair), budget, strategy, stride, n_special, cnt.ctypes.data, ctypes.byref(mx),
                                  ctypes.byref(err), ctypes.byref(sm))
    if err.value & 32:
        return "too short to respect"
    if err.value & 64:
        return f"must be strictly less than `max_len={sm.value}`"
    W = mx.value
    seg, sp = [[], [], []], 0
    b_first, tx, ty = 0, 0, 0
    for kind, v, t in pieces:
        if kind == "seq":
            if sp == 0:
                b_first, tx = int(v == 1), t
            else:
                ty = t
            sp += 1
        else:
            seg[sp].append(v | t << 24 if is_pair else v)
    special = np.asarray(seg[0] + seg[1] + seg[2] + [0], dtype=np.uint32)
    out = np.zeros((R, W), np.uint32); tout = np.zeros((R, W), np.uint8); mask = np.zeros((R, W), np.uint8)
    olen = np.zeros(R + 1, np.uint32); samp = np.zeros(R + 1, np.uint32); ooff = np.zeros((R, W, 2), np.uint32)
    L.b2t_emul_overflow_rows(ids.ctypes.data, offs.ctypes.data, rp.ctypes.data, n_in, int(is_pair), cnt.ctypes.data, R, W, budget, strategy, stride,
                             int(left), int(pad_left), 7, 5, len(seg[0]), len(seg[1]), len(seg[2]), special.ctypes.data, b_first, tx, ty,
                             overflow_types[0], overflow_types[1], 0, out.ctypes.data, tout.ctypes.data, mask.ctypes.data, olen.ctypes.data,
                             samp.ctypes.data, ooff.ctypes.data)
    return out, tout, mask, olen[:R], samp[:R], ooff


def restated_rows(lens, is_pair, pieces, budget, strategy, stride, left, overflow_type=None):
    """the same batch through the shim's host restatement (pairs.post_process), padded to the longest row of all;
    overflow_type: the type id a RobertaProcessing-style template gives every overflowing part"""
    rp = np.zeros(len(lens) + 1, dtype=np.int64); np.cumsum(lens, out=rp[1:])
    ids = np.concatenate([1000 * d + np.arange(n) for d, n in enumerate(lens)] + [np.zeros(0)]).astype(np.uint32)
    offs = np.concatenate([np.stack([np.arange(n), np.arange(n) + 1], axis=1) for n in lens] + [np.zeros((0, 2))]).astype(np.uint32)
    single = [p for p in pieces if p[0] == "special" or p[1] == 0] if not is_pair else None
    tpl = {"pair": pieces, "single": single, "trim": None, "pre": [], "post": [], "overflow_type": overflow_type}
    tr = dict(max_length=budget + sum(1 for p in (pieces if is_pair else single) if p[0] == "special"), stride=stride,
              strategy=strategy, direction="left" if left else "right")
    return oo.dense_overflow_rows(ids, offs, rp, is_pair=is_pair, template=tpl, truncation=tr,
                                  padding=dict(length=None, direction="right", pad_id=7, pad_type_id=5), add_special_tokens=True, pad_all_rows=True)


NS = (0, 1, 2, 5, 13, 40)


@pytest.mark.parametrize("order", list(EMUL_TEMPLATES))
def test_overflow_kernels_match_post_process(order):
    """the count pass, the row-sample pass and the OVER + OFFS row kernels, run on the host, == pairs.post_process on
    batches of every (n1, n2) of NS, for every budget in [0, 48], strides 0, 1, budget / 2, budget - 1 and budget, every
    strategy and both directions (the stride panic and SequenceTooShort included); single sequences likewise"""
    L = _emul()
    pieces = EMUL_TEMPLATES[order]
    lens = [n for a in NS for b in NS for n in (a, b)]
    for budget in range(49):
        for stride in sorted({0, 1, budget // 2, max(budget - 1, 0), budget}):
            for strategy in range(3):
                for left in (False, True):
                    what = (order, budget, stride, STRATEGIES[strategy], left)
                    got = emul_rows(L, lens, True, pieces, budget, strategy, stride, left, (0, 1))
                    same(got, restated_rows(lens, True, pieces, budget, STRATEGIES[strategy], stride, left), what)
                    if strategy == 0 and order == "a_first":
                        single = [p for p in pieces if p[0] == "special" or p[1] == 0][:2]   # pre A post
                        same(emul_rows(L, list(range(41)), False, single, budget, 0, stride, left, (0, 0)),
                             restated_rows(list(range(41)), False, single, budget, "longest_first", stride, left), what + ("single",), is_pair=False)


def test_overflow_type_ids_follow_the_roberta_rule():
    """overflow types (0, 0), as the shim passes them under RobertaProcessing with special tokens: every row, type ids
    included, == pairs.post_process with the template's overflow_type rule"""
    L = _emul()
    lens = [n for a in (0, 3, 17, 40) for b in (0, 5, 29, 40) for n in (a, b)]
    for order, pieces in EMUL_TEMPLATES.items():
        for budget, stride, strategy in ((20, 3, 0), (30, 7, 0), (25, 2, 2), (25, 4, 1), (9, 0, 0)):
            for left in (False, True):
                got = emul_rows(L, lens, True, pieces, budget, strategy, stride, left, (0, 0))
                exp = restated_rows(lens, True, pieces, budget, STRATEGIES[strategy], stride, left, overflow_type=0)
                same(got, exp, (order, budget, stride, strategy, left))
                if not isinstance(exp, str):
                    assert exp[0].shape[0] > len(lens) // 2 and 0 in exp[1][1:, 1].tolist()   # (overflowing rows do exist)


def test_count_pass_exhaustive():
    """dense_count_kernel == truncation_spans composed with pairs.truncate_pair (the max_len each sequence of a pair is cut
    to) for every n1, n2 in [0, 40], every budget in [0, 48], every stride in [0, budget] and every strategy: the rows of
    every input, the longest row, SequenceTooShort and the stride panic (with the max_len it names); single sequences for
    every n in [0, 40] likewise"""
    L = _emul()
    N, M = 41, 49
    # parts and longest part of a sequence of n tokens cut to max_len m with stride s (0 parts: the reference panics)
    cnt = np.zeros((N, M, M), np.int64); mx = np.zeros((N, M, M), np.int64)
    for n in range(N):
        for m in range(M):
            for st in range(M):
                try:
                    sp = truncation_spans(n, m, st, "right")
                except ValueError:
                    continue
                cnt[n, m, st], mx[n, m, st] = len(sp), max(b - a for a, b in sp)
    n1, n2 = (x.reshape(-1) for x in np.meshgrid(np.arange(N), np.arange(N), indexing="ij"))
    rp = np.zeros(2 * n1.size + 1, np.uint64); np.cumsum(np.stack([n1, n2], 1).reshape(-1), out=rp[1:])
    rps = np.zeros(N + 1, np.uint64); np.cumsum(np.arange(N), out=rps[1:])
    out = np.zeros(n1.size + 1, np.uint32)
    m_all, err, sm = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
    real_truncate = shim_pairs.truncate
    for budget in range(M):
        for strategy in range(3):
            # the max_len truncate_pair gives each sequence (its length when it is not cut); None: SequenceTooShort
            m1, m2, short = n1.copy(), n2.copy(), np.zeros(n1.size, bool)
            for k in range(n1.size):
                a, b = shim_pairs.PE([0] * int(n1[k])), shim_pairs.PE([0] * int(n2[k]))
                cut = {}
                shim_pairs.truncate = lambda pe, max_len, stride, direction: cut.__setitem__(id(pe), max_len)
                try:
                    shim_pairs.truncate_pair(a, b, dict(max_length=budget, stride=0, direction="right", strategy=STRATEGIES[strategy]))
                    m1[k], m2[k] = cut.get(id(a), n1[k]), cut.get(id(b), n2[k])
                except ValueError:
                    short[k] = True
                finally:
                    shim_pairs.truncate = real_truncate
            m1c, m2c = np.minimum(m1, M - 1), np.minimum(m2, M - 1)   # (a max_len above n keeps the sequence: same as n)
            for stride in range(budget + 1):
                p1, p2 = cnt[n1, m1c, stride], cnt[n2, m2c, stride]
                panic = ~short & ((p1 == 0) | (p2 == 0))
                ok = ~short & ~panic
                R = L.b2t_emul_overflow_count(rp.ctypes.data, n1.size, 1, budget, strategy, stride, 3, out.ctypes.data, ctypes.byref(m_all),
                                              ctypes.byref(err), ctypes.byref(sm))
                what = (budget, strategy, stride)
                assert bool(err.value & 32) == bool(short.any()) and bool(err.value & 64) == bool(panic.any()), what
                assert np.array_equal(out[:n1.size][ok], (p1 * p2)[ok]), what
                if panic.any():
                    assert sm.value == int(np.where(p1 == 0, m1, m2)[panic].max()), what
                if not short.any() and not panic.any():
                    assert R == int((p1 * p2).sum()) and m_all.value == int((3 + mx[n1, m1c, stride] + mx[n2, m2c, stride]).max()), what
                if strategy == 0:   # single sequences: each cut to the budget itself
                    ns = np.arange(N)
                    R = L.b2t_emul_overflow_count(rps.ctypes.data, N, 0, budget, 0, stride, 2, out.ctypes.data, ctypes.byref(m_all),
                                                  ctypes.byref(err), ctypes.byref(sm))
                    ps = cnt[ns, budget, stride]
                    pan = ps == 0
                    assert bool(err.value & 64) == bool(pan.any()) and not err.value & 32, what
                    assert np.array_equal(out[:N][~pan], ps[~pan]), what
                    if not pan.any():
                        assert m_all.value == int((2 + mx[ns, budget, stride]).max()), what


@pytest.mark.skipif(tk is None, reason="reference wheel not importable")
@pytest.mark.parametrize("name", list(tdp.TEMPLATES))
def test_overflow_oracle_matches_wheel(name):
    """the restatement == the wheel on every template and setting (offsets where the post-processor does not trim them:
    offset rows are refused there)"""
    js = tdp.tokenizer_json(name)
    for key, tr, pd, is_pair, ast in cases():
        tr = resolve(js, tr, is_pair, ast)
        inputs = arrange(inputs_for(11), tr, is_pair)
        o = oracle_rows(js, inputs, tr, pd, is_pair, ast)
        same(o, wheel_rows(js, inputs, tr, pd, ast), (name, key), is_pair, not trimmed(name), ref=o)


@pytest.mark.parametrize("name", list(tdp.TEMPLATES))
def test_overflow_oracle_matches_golden(name):
    """the restatement against committed vectors of the wheel (no wheel needed)"""
    g = _golden()
    js = tdp.tokenizer_json(name)
    for key, tr, pd, is_pair, ast in cases():
        tr = resolve(js, tr, is_pair, ast)
        inputs = arrange([tuple(p) for p in g["inputs"]], tr, is_pair)
        o = oracle_rows(js, inputs, tr, pd, is_pair, ast)
        same(o, golden_rows(g["cases"][f"{name}/{key}"]), (name, key), is_pair, not trimmed(name), ref=o)


def _apply(tok, tr, pd):
    tdp._apply(tok, tr, pd)


def test_overflow_spec_fields_and_refusals():
    from tokenizers_b200 import UnsupportedConfig, _lib
    tok = helpers.oracle_backed_tokenizer(tdp.tokenizer_json("roberta"))
    _apply(tok, dict(max_length=32, strategy="only_second", direction="right", stride=4), tdp.SETTINGS[0][1])
    sp, _ = tok.pair_dense_spec(return_overflowing_tokens=True)
    assert (sp.stride, sp.dense_flags, sp.overflow_type_a, sp.overflow_type_b) == (4, _lib.DENSE_OVERFLOW, 0, 0)
    sp, _ = tok.pair_dense_spec(add_special_tokens=False, return_overflowing_tokens=True)
    assert (sp.overflow_type_a, sp.overflow_type_b) == (0, 1)
    with pytest.raises(UnsupportedConfig):   # offsets behind trim_offsets
        tok.pair_dense_spec(return_overflowing_tokens=True, return_offsets_mapping=True)
    with pytest.raises(UnsupportedConfig):   # a stride without overflowing parts: unchanged
        tok.pair_dense_spec()
    sp, _ = tok.dense_spec(return_overflowing_tokens=True)
    assert (sp.stride, sp.dense_flags) == (4, _lib.DENSE_OVERFLOW)
    sp, _ = tok.dense_spec()
    assert (sp.stride, sp.dense_flags, ctypes.sizeof(sp)) == (0, 0, 72) and ctypes.sizeof(_lib.PairDenseSpec) == 80
    tok = helpers.oracle_backed_tokenizer(tdp.tokenizer_json("bert"))
    _apply(tok, dict(max_length=32, strategy="longest_first", direction="right", stride=4), tdp.SETTINGS[0][1])
    sp, _ = tok.pair_dense_spec(return_overflowing_tokens=True, return_offsets_mapping=True)
    assert (sp.dense_flags, sp.overflow_type_a, sp.overflow_type_b) == (_lib.DENSE_OVERFLOW | _lib.DENSE_OFFSETS, 0, 1)
    _apply(tok, dict(max_length=0, strategy="longest_first", direction="right", stride=0), tdp.SETTINGS[0][1])
    with pytest.raises(UnsupportedConfig):   # truncation to max_length 0: still no dense form
        tok.dense_spec(return_overflowing_tokens=True)


# ------------------------------------------------------------------------------------------------------------- GPU
def engine_rows(tok, inputs, tr, pd, is_pair, ast=True, offsets=True):
    from tokenizers_b200 import B2TError
    _apply(tok, tr, pd)
    try:
        f = tok.encode_pairs_dense if is_pair else tok.encode_batch_dense
        out = f(inputs, add_special_tokens=ast, return_overflowing_tokens=True, return_offsets_mapping=offsets)
    except ValueError as ex:
        if PANIC not in str(ex) and TOO_SHORT not in str(ex):
            raise
        return str(ex)
    except B2TError as ex:
        if NOT_FIT not in str(ex):
            raise
        return str(ex)
    return (out["input_ids"], out.get("token_type_ids"), out["attention_mask"], out["lengths"], out["overflow_to_sample_mapping"],
            out.get("offset_mapping"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(tdp.TEMPLATES))
def test_gpu_overflow_matches_oracle_wheel_and_golden(name):
    from tokenizers_b200 import Tokenizer
    js = tdp.tokenizer_json(name)
    tok = Tokenizer.from_str(js)
    g = _golden()
    offs = not trimmed(name)
    for key, tr, pd, is_pair, ast in cases():
        tr = resolve(js, tr, is_pair, ast)
        inputs, ginputs = arrange(inputs_for(12), tr, is_pair), arrange([tuple(p) for p in g["inputs"]], tr, is_pair)
        got = engine_rows(tok, inputs, tr, pd, is_pair, ast, offs)
        o = oracle_rows(js, inputs, tr, pd, is_pair, ast)
        same(got, o, (name, key, "oracle"), is_pair, offs)
        if tk is not None:
            same(got, wheel_rows(js, inputs, tr, pd, ast), (name, key, "wheel"), is_pair, offs, ref=o)
        same(engine_rows(tok, ginputs, tr, pd, is_pair, ast, offs), golden_rows(g["cases"][f"{name}/{key}"]), (name, key, "golden"), is_pair, offs,
             ref=oracle_rows(js, ginputs, tr, pd, is_pair, ast))


def qa_inputs():
    """questions with corpus contexts: pairs around 64 KiB chunk edges, a context larger than a chunk (hundreds of
    windows), and enough windows in all to grow the pinned rows past their first guess (one row per input)"""
    data, off = corpus.generate(2, 33, 0, 600)
    docs = corpus.to_strings(data, off)
    qs = ["what is " + " ".join(d.split()[:3]) for d in docs]
    pairs = list(zip(qs, docs))
    filler = "lorem ipsum dolor sit amet, consectetur adipiscing elit "
    pairs.append(("where is the end?", (filler * 2000)[:90000]))
    return pairs + list(zip(qs[::-1], docs[::-1]))[:100]


@pytest.mark.gpu
def test_gpu_overflow_chunks_growth_and_device_entry_points(monkeypatch):
    from tokenizers_b200 import Tokenizer, _lib
    import torch
    js = tdp.tokenizer_json("bert")
    pairs = qa_inputs()
    tr, pd = dict(max_length=64, stride=16, strategy="only_second", direction="right"), dict(length=64, direction="right", pad_id=0, pad_type_id=0)
    exp = oracle_rows(js, pairs, tr, pd, True, True)
    assert not isinstance(exp, str) and len(exp[4]) > 4 * len(pairs) and np.bincount(exp[4]).max() > 300
    monkeypatch.setenv("B2T_CHUNK_BYTES", "65536")   # many chunks, each with its own number of rows
    tok = Tokenizer.from_str(js)
    same(engine_rows(tok, pairs, tr, pd, True), exp, "fixed length, 64 KiB chunks")
    tr1, pd1 = dict(max_length=48, stride=8, strategy="longest_first", direction="left"), dict(length=None, direction="left", pad_id=0, pad_type_id=1)
    singles = [b for _, b in pairs]
    exp1 = oracle_rows(js, singles, tr1, pd1, False, True)
    same(engine_rows(tok, singles, tr1, pd1, False), exp1, "single sequences, BatchLongest", is_pair=False)
    L = _lib.lib()
    cudart = ctypes.CDLL("libcudart.so")

    def dev(ptr, count, dtype):
        out = np.empty(count, dtype=dtype)
        if count:
            assert cudart.cudaMemcpy(ctypes.c_void_p(out.ctypes.data), ctypes.c_void_p(ptr), ctypes.c_size_t(out.nbytes), 2) == 0
        return out
    for is_pair, seqs, trd, pdd, e in ((True, pairs, tr, pd, exp), (False, singles, tr1, pd1, exp1)):
        _apply(tok, trd, pdd)
        sp, keep = (tok.pair_dense_spec if is_pair else tok.dense_spec)(return_overflowing_tokens=True, return_offsets_mapping=True)
        data, off = helpers.pack_docs(flat(seqs))
        d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        res = ctypes.c_void_p()
        f = L.b2t_encode_pairs_dense_device if is_pair else L.b2t_encode_batch_dense_device
        _lib.check(f(tok.handle, d_bytes.data_ptr(), len(data), d_off.data_ptr(), len(seqs), ctypes.byref(sp), None, ctypes.byref(res)))
        torch.cuda.synchronize()
        W, R = L.b2t_result_dense_length(res), L.b2t_result_dense_rows(res)
        assert L.b2t_result_on_device(res) == 1 and L.b2t_result_n_docs(res) == len(seqs) and (R, W) == e[0].shape
        got = (dev(L.b2t_result_dense_ids(res), R * W, np.uint32).reshape(R, W),
               dev(L.b2t_result_type_ids(res), R * W, np.uint8).reshape(R, W) if is_pair else None,
               dev(L.b2t_result_attention_mask(res), R * W, np.uint8).reshape(R, W), dev(L.b2t_result_row_lengths(res), R, np.uint32),
               dev(L.b2t_result_row_sample(res), R, np.uint32), dev(L.b2t_result_dense_offsets(res), 2 * R * W, np.uint32).reshape(R, W, 2))
        L.b2t_result_free(res)
        same(got, e, ("device entry point", is_pair), is_pair)


@pytest.mark.gpu
def test_gpu_overflow_bert_pipeline_and_device_added_tokens():
    from tokenizers_b200 import Tokenizer
    # the bert-base pipeline: offsets mapped back through BertNormalizer
    j = json.loads(helpers.bert_json(helpers.BERT_UNCASED))
    j["post_processor"] = tdp.TEMPLATES["bert"][1](j["model"]["vocab"])
    js = json.dumps(j)
    tok = Tokenizer.from_str(js)
    for tr, pd in SETTINGS[:4]:
        for is_pair in (True, False):
            if not is_pair and tr["strategy"] == "only_second":
                continue
            inputs = arrange([(a.upper() + " Àé 中文 naïve", b) for a, b in inputs_for(21)], tr, is_pair)
            got = engine_rows(tok, inputs, tr, pd, is_pair)
            o = oracle_rows(js, inputs, tr, pd, is_pair, True)
            same(got, o, ("bert", tr, is_pair), is_pair)
            if tk is not None:
                same(got, wheel_rows(js, inputs, tr, pd, True), ("bert", tr, is_pair, "wheel"), is_pair, ref=o)
    # added tokens extracted on the device, inside both sequences (offset rows: no trimming post-processor here)
    js = json.loads(helpers.with_added_tokens(helpers.asset_json("wordpiece")))
    js["post_processor"] = tdp.TEMPLATES["bert"][1](js["model"]["vocab"])
    js = json.dumps(js)
    tok, ref = Tokenizer.from_str(js), helpers.oracle_backed_tokenizer(js)
    assert tok._dev_added
    docs = helpers.added_token_docs(5, 300)
    pairs = list(zip(docs[0::2], docs[1::2]))
    data, off = helpers.pack_docs(flat(pairs))
    be, _ = ref._encode_core(data, off, 1, True)   # (WANT_OFFSETS)
    tr, pd = dict(max_length=24, stride=3, strategy="longest_first", direction="right"), dict(length=None, direction="right", pad_id=0, pad_type_id=1)
    got = engine_rows(tok, pairs, tr, pd, True)
    exp = oo.dense_overflow_rows(be.ids, be.offsets, be.row_ptr, is_pair=True, template=parse_post_processor(json.loads(js)["post_processor"]),
                                 truncation=tr, padding=pd, add_special_tokens=True)
    same(got, exp, "device added tokens")
    if tk is not None:
        same(got, wheel_rows(js, pairs, tr, pd, True), "device added tokens, wheel", ref=exp)


def device_rows(tok, seqs, is_pair, sp):
    """b2t_encode_pairs_dense_device / b2t_encode_batch_dense_device with the spec sp -> (ids, type ids | None, mask,
    lengths, sample | None, offsets | None) copied back from the device"""
    from tokenizers_b200 import _lib
    import torch
    L = _lib.lib()
    cudart = ctypes.CDLL("libcudart.so")

    def dev(ptr, count, dtype):
        out = np.empty(count, dtype=dtype)
        if count:
            assert cudart.cudaMemcpy(ctypes.c_void_p(out.ctypes.data), ctypes.c_void_p(ptr), ctypes.c_size_t(out.nbytes), 2) == 0
        return out
    data, off = helpers.pack_docs(flat(seqs))
    d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    res = ctypes.c_void_p()
    f = L.b2t_encode_pairs_dense_device if is_pair else L.b2t_encode_batch_dense_device
    _lib.check(f(tok.handle, d_bytes.data_ptr(), len(data), d_off.data_ptr(), len(seqs), ctypes.byref(sp), None, ctypes.byref(res)))
    torch.cuda.synchronize()
    W, R = L.b2t_result_dense_length(res), L.b2t_result_dense_rows(res)
    assert L.b2t_result_on_device(res) == 1 and L.b2t_result_n_docs(res) == len(seqs)
    sample, offs = L.b2t_result_row_sample(res), L.b2t_result_dense_offsets(res)
    got = (dev(L.b2t_result_dense_ids(res), R * W, np.uint32).reshape(R, W),
           dev(L.b2t_result_type_ids(res), R * W, np.uint8).reshape(R, W) if is_pair else None,
           dev(L.b2t_result_attention_mask(res), R * W, np.uint8).reshape(R, W), dev(L.b2t_result_row_lengths(res), R, np.uint32),
           dev(sample, R, np.uint32) if sample else None, dev(offs, 2 * R * W, np.uint32).reshape(R, W, 2) if offs else None)
    L.b2t_result_free(res)
    return got


@pytest.mark.gpu
def test_gpu_offsets_without_overflow(monkeypatch):
    """return_offsets_mapping alone: the kept rows with their offsets (the <0, 1> row kernels), == the restatement's kept
    rows -- on the host path (a fixed length in 64 KiB chunks, and BatchLongest) and on both device entry points, each
    right after an overflow + offsets call on the same engine (whose offset buffers then hold other rows)"""
    from tokenizers_b200 import Tokenizer
    monkeypatch.setenv("B2T_CHUNK_BYTES", "65536")
    js = tdp.tokenizer_json("bert")
    tok = Tokenizer.from_str(js)
    qa = qa_inputs()
    for is_pair in (True, False):
        seqs = qa if is_pair else [b for _, b in qa]
        strategy = "only_second" if is_pair else "longest_first"
        for tr, pd in ((dict(max_length=64, stride=0, strategy=strategy, direction="right"), dict(length=64, direction="right", pad_id=0, pad_type_id=0)),
                       (dict(max_length=48, stride=0, strategy=strategy, direction="left"), dict(length=None, direction="left", pad_id=0, pad_type_id=1))):
            full = oracle_rows(js, seqs, tr, pd, is_pair, True)
            assert not isinstance(full, str)
            kept = np.r_[True, np.diff(full[4].astype(np.int64)) != 0]
            assert kept.sum() == len(seqs) and not kept.all()   # (the stride-0 truncation does make overflowing rows)
            exp = tuple(None if k == 4 else x[kept] for k, x in enumerate(full))
            what = (is_pair, tr["direction"])
            # host path
            assert not isinstance(engine_rows(tok, seqs, dict(tr, stride=8), pd, is_pair), str)
            _apply(tok, tr, pd)
            out = (tok.encode_pairs_dense if is_pair else tok.encode_batch_dense)(seqs, return_offsets_mapping=True)
            assert "overflow_to_sample_mapping" not in out and out["offset_mapping"].shape == exp[0].shape + (2,)
            same((out["input_ids"], out.get("token_type_ids"), out["attention_mask"], out["lengths"], None, out["offset_mapping"]), exp,
                 what + ("host",), is_pair)
            # device entry points
            _apply(tok, dict(tr, stride=8), pd)
            spec = tok.pair_dense_spec if is_pair else tok.dense_spec
            sp, keep = spec(return_overflowing_tokens=True, return_offsets_mapping=True)
            assert device_rows(tok, seqs, is_pair, sp)[4] is not None
            _apply(tok, tr, pd)
            sp, keep = spec(return_offsets_mapping=True)
            got = device_rows(tok, seqs, is_pair, sp)
            assert got[4] is None and got[5] is not None
            same(got, exp, what + ("device",), is_pair)


@pytest.mark.gpu
def test_gpu_overflow_refusals_empty_batch_old_spec_and_switches_off():
    from tokenizers_b200 import Tokenizer, UnsupportedConfig, B2TError, _lib
    js = tdp.tokenizer_json("bert")
    tok = Tokenizer.from_str(js)
    pairs = inputs_for(13)
    # a whole sequence overflows (budget 1 under longest_first cuts the shorter one to 0): longer than L, refused
    _apply(tok, dict(max_length=4, stride=0, strategy="longest_first", direction="right"), dict(length=None, direction="right", pad_id=0, pad_type_id=0))
    with pytest.raises(B2TError, match="does not fit") as ei:
        tok.encode_pairs_dense(pairs, return_overflowing_tokens=True)
    assert ei.value.code == _lib.B2T_ERR_INVALID
    assert "fit" in oracle_rows(js, pairs, dict(max_length=4, stride=0, strategy="longest_first", direction="right"),
                                dict(length=None, direction="right", pad_id=0, pad_type_id=0), True, True)
    # the stride panic, with the reference's message: B is cut to 10 - 3 special tokens - the tokens of A, not more than
    # the stride
    _apply(tok, dict(max_length=10, stride=7, strategy="only_second", direction="right"), tdp.SETTINGS[0][1])
    m = 10 - 3 - len(orc.Oracle(js).encode_batch(["why"])[0])
    with pytest.raises(ValueError, match=f"strictly less than `max_len={m}`"):
        tok.encode_pairs_dense([("why", " ".join(tdp.WORDS * 3))], return_overflowing_tokens=True)
    # offsets behind a trimming post-processor
    rt = Tokenizer.from_str(tdp.tokenizer_json("roberta"))
    _apply(rt, dict(max_length=32, stride=4, strategy="only_second", direction="right"), tdp.SETTINGS[0][1])
    long_second = tdp.arrange(pairs, dict(strategy="only_second"))   # (the sequence only_second cuts is the long one)
    with pytest.raises(UnsupportedConfig):
        rt.encode_pairs_dense(long_second, return_overflowing_tokens=True, return_offsets_mapping=True)
    assert rt.encode_pairs_dense(long_second, return_overflowing_tokens=True)["input_ids"].shape[0] > len(pairs)
    # an empty batch
    _apply(tok, dict(max_length=32, stride=4, strategy="only_second", direction="right"), tdp.SETTINGS[0][1])
    got = tok.encode_pairs_dense([], return_overflowing_tokens=True, return_offsets_mapping=True)
    assert got["input_ids"].shape == (0, 40) and got["overflow_to_sample_mapping"].shape == (0,) and got["offset_mapping"].shape == (0, 40, 2)
    got = tok.encode_batch_dense([], return_overflowing_tokens=True)
    assert got["input_ids"].shape == (0, 40) and got["overflow_to_sample_mapping"].shape == (0,)
    # both switches off: the calls and their dicts as they were; an old-size spec gives byte-identical rows
    L = _lib.lib()
    for is_pair in (True, False):
        _apply(tok, dict(max_length=32, stride=0, strategy="longest_first", direction="left"), dict(length=None, direction="right", pad_id=0, pad_type_id=0))
        seqs = pairs if is_pair else [a for a, _ in pairs]
        plain = (tok.encode_pairs_dense if is_pair else tok.encode_batch_dense)(seqs)
        assert set(plain) == ({"input_ids", "token_type_ids", "attention_mask", "lengths"} if is_pair else {"input_ids", "attention_mask", "lengths"})
        over = (tok.encode_pairs_dense if is_pair else tok.encode_batch_dense)(seqs, return_overflowing_tokens=True)
        kept = np.r_[True, np.diff(over["overflow_to_sample_mapping"].astype(np.int64)) != 0]
        for k in plain:
            assert np.array_equal(over[k][kept], plain[k]), (is_pair, k)
        data, off = helpers.pack_docs(flat(seqs))
        outs = []
        for size in (None, 64):
            sp, keep = (tok.pair_dense_spec if is_pair else tok.dense_spec)()
            if size:
                sp.struct_size, sp.stride, sp.dense_flags = size, 7, 3   # (fields past the old size must be ignored)
            res = ctypes.c_void_p()
            f = L.b2t_encode_pairs_dense if is_pair else L.b2t_encode_batch_dense
            _lib.check(f(tok.handle, data.ctypes.data, off.ctypes.data, len(seqs), ctypes.byref(sp), ctypes.byref(res)))
            R, W = L.b2t_result_dense_rows(res), L.b2t_result_dense_length(res)
            assert R == L.b2t_result_n_docs(res) == len(seqs) and not L.b2t_result_row_sample(res) and not L.b2t_result_dense_offsets(res)
            outs.append(bytes(np.ctypeslib.as_array(ctypes.cast(L.b2t_result_dense_ids(res), ctypes.POINTER(ctypes.c_uint8)), shape=(R * W * 4,))))
            L.b2t_result_free(res)
        assert outs[0] == outs[1] and outs[0] == plain["input_ids"].tobytes()
