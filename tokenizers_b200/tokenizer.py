"""Host-side mirror of the reference's Python surface for the encode_batch path.

Mirrors `tokenizers.Tokenizer` (bindings/python/src/tokenizer.rs:510-1461 in the reference tree): `from_file`,
`from_str`, `encode`, `encode_batch`, `encode_batch_fast`, `token_to_id`, `id_to_token`, `get_vocab_size`, and
`tokenizers.Encoding` (bindings/python/src/encoding.rs:133-225): `ids`, `tokens`, `offsets`, `word_ids`, `type_ids`,
`attention_mask`, `special_tokens_mask`.  All tokenization happens in libb2t.so on the GPU; configurations outside the
hot path raise `UnsupportedConfig` (there is no CPU fallback).  The two host steps the reference runs around the path are
mirrored here: added-token extraction before it (`added.py`) and the special-token template after it (`post_process`).
"""
import ctypes, json
import numpy as np
from . import _lib, added
from ._lib import B2TError

LLAMA3_PATTERN = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*"
                  r"|\s*[\r\n]+|\s+(?!\S)|\s+")


class UnsupportedConfig(ValueError):
    """The tokenizer.json asks for something outside the accelerated path (the reference handles it on CPU)."""


def _pack(strings, off_dtype):
    """list of str -> (their UTF-8 bytes back to back as uint8 (a read-only view of one bytes object), off_dtype[n + 1]
    offsets).  Raises AttributeError for an element that is not a str."""
    bs = [s.encode("utf-8") for s in strings]
    off = np.zeros(len(bs) + 1, dtype=off_dtype)
    if bs:
        np.cumsum(np.fromiter(map(len, bs), dtype=np.int64, count=len(bs)), out=off[1:])
    return np.frombuffer(b"".join(bs), dtype=np.uint8), off


def parse_post_processor(pp):
    """post_processor of tokenizer.json -> None (nothing to do) or
    {"pre": [(id, type_id)], "post": [...], "type_id": t, "trim": None | add_prefix_space, "single": pieces, "pair": pieces}
    (processors/template.rs:646-, processors/bert.rs, processors/roberta.rs, processors/sequence.rs;
    "trim": ByteLevel / Roberta `trim_offsets`, pre_tokenizers/byte_level.rs:174-234).  pre / post / type_id describe
    the single-sequence template for the vectorised CSR path; `single` / `pair` are the same templates as piece lists
    [("seq", 0 | 1, type_id) | ("special", token id, type_id)] for the per-input path that handles pairs."""
    if pp is None:
        return None
    ty = pp.get("type")

    def from_pieces(single, pair, trim):
        pre, post, seen, seq_type = [], [], False, 0
        for kind, v, t in single:
            if kind == "seq":
                seen, seq_type = True, t
            else:
                (post if seen else pre).append((v, t))
        return {"pre": pre, "post": post, "type_id": seq_type, "trim": trim, "single": single, "pair": pair}

    plain = ([("seq", 0, 0)], [("seq", 0, 0), ("seq", 1, 1)])
    if ty == "ByteLevel":
        return from_pieces(plain[0], plain[1], bool(pp.get("add_prefix_space", True))) if pp.get("trim_offsets", True) else None
    if ty == "Sequence":
        out = None
        for sub in pp.get("processors", []):
            t = parse_post_processor(sub)
            if t is None:
                continue
            if out is None:
                out = t
            elif (out["pre"] or out["post"]) and (t["pre"] or t["post"] or t["trim"] is not None):
                raise UnsupportedConfig("post-processor Sequence: only [offset trimming, one special-token template] in that order")
            else:
                out = dict(t, trim=out["trim"] if t["trim"] is None else t["trim"])
        return out
    if ty in ("BertProcessing", "RobertaProcessing"):
        cls, sep = int(pp["cls"][1]), int(pp["sep"][1])
        if ty == "BertProcessing":
            single = [("special", cls, 0), ("seq", 0, 0), ("special", sep, 0)]
            pair = single + [("seq", 1, 1), ("special", sep, 1)]
            return from_pieces(single, pair, None)
        trim = bool(pp.get("add_prefix_space", True)) if pp.get("trim_offsets", True) else None
        single = [("special", cls, 0), ("seq", 0, 0), ("special", sep, 0)]
        pair = single + [("special", sep, 0), ("seq", 1, 0), ("special", sep, 0)]
        return dict(from_pieces(single, pair, trim), overflow_type=0)  # roberta.rs: type id 0 everywhere, overflowing parts too
    if ty == "TemplateProcessing":
        def pieces(tpl):
            out, seen = [], set()
            for piece in tpl:
                if "Sequence" in piece:
                    i = 0 if piece["Sequence"].get("id") == "A" else 1
                    if i in seen:
                        raise UnsupportedConfig("a template may use each sequence once")
                    seen.add(i)
                    out.append(("seq", i, int(piece["Sequence"].get("type_id", 0))))
                else:
                    sp = piece["SpecialToken"]
                    out.extend(("special", int(i), int(sp.get("type_id", 0))) for i in pp["special_tokens"][sp["id"]]["ids"])
            return out, seen
        single, seen1 = pieces(pp.get("single", []))
        pair, seen2 = pieces(pp.get("pair", []))
        if seen1 != {0}:
            raise UnsupportedConfig("TemplateProcessing.single must contain sequence A exactly once")
        return from_pieces(single, pair if seen2 == {0, 1} else None, None)
    raise UnsupportedConfig(f"post-processor {ty} is not supported")


def parse_truncation(t):
    """tokenizer.json `truncation` (utils/truncation.rs:42-58) -> dict with the Python binding's spelling, or None"""
    if t is None:
        return None
    strategy = {"LongestFirst": "longest_first", "OnlyFirst": "only_first", "OnlySecond": "only_second"}[t.get("strategy", "LongestFirst")]
    return {"max_length": int(t["max_length"]), "stride": int(t.get("stride", 0)), "strategy": strategy,
            "direction": t.get("direction", "Right").lower()}


def parse_padding(p):
    """tokenizer.json `padding` (utils/padding.rs:21-48) -> dict with the Python binding's spelling, or None"""
    if p is None:
        return None
    st = p.get("strategy", "BatchLongest")
    return {"length": None if st == "BatchLongest" else int(st["Fixed"]), "direction": p.get("direction", "Right").lower(),
            "pad_to_multiple_of": p.get("pad_to_multiple_of"), "pad_id": int(p.get("pad_id", 0)),
            "pad_type_id": int(p.get("pad_type_id", 0)), "pad_token": p.get("pad_token", "[PAD]")}


def parse_tokenizer_json(js):
    """tokenizer.json (tokenizer/serialization.rs:15-48 in the reference) -> engine configuration dict."""
    nz, norm = js.get("normalizer"), 0
    if nz is not None:
        # normalizers/bert.rs:52-136; every other normalizer stays outside the accelerated path
        if nz.get("type") != "BertNormalizer":
            raise UnsupportedConfig(f"normalizer {nz.get('type')} is not on the accelerated path (BertNormalizer is)")
        lower = bool(nz.get("lowercase", True))
        strip = lower if nz.get("strip_accents") is None else bool(nz["strip_accents"])   # bert.rs:128
        norm = (_lib.NORM_BERT | (_lib.NORM_CLEAN_TEXT if nz.get("clean_text", True) else 0) | (_lib.NORM_CHINESE_CHARS if nz.get("handle_chinese_chars", True) else 0) |
                (_lib.NORM_STRIP_ACCENTS if strip else 0) | (_lib.NORM_LOWERCASE if lower else 0))
    template = parse_post_processor(js.get("post_processor"))
    pt, m = js.get("pre_tokenizer"), js["model"]
    cfg = dict(add_prefix_space=0, ignore_merges=0, unk=None, prefix="##", max_chars=100, merges=[], normalizer=norm)
    if pt is None:
        raise UnsupportedConfig("a pre_tokenizer is required")
    if pt["type"] == "ByteLevel":
        cfg["pretok"] = _lib.PRETOK_BYTELEVEL if pt.get("use_regex", True) else _lib.PRETOK_BYTELEVEL_NOREGEX
        cfg["add_prefix_space"] = int(pt.get("add_prefix_space", True))
    elif pt["type"] == "Whitespace":
        cfg["pretok"] = _lib.PRETOK_WHITESPACE
    elif pt["type"] == "BertPreTokenizer":
        cfg["pretok"] = _lib.PRETOK_BERT
    elif pt["type"] == "Sequence" and len(pt.get("pretokenizers", [])) == 2:
        a, b = pt["pretokenizers"]
        ok = (a.get("type") == "Split" and a.get("pattern", {}).get("Regex") == LLAMA3_PATTERN and a.get("behavior") == "Isolated"
              and not a.get("invert", False) and b.get("type") == "ByteLevel" and not b.get("use_regex", True)
              and not b.get("add_prefix_space", True))
        if not ok:
            raise UnsupportedConfig("only Sequence[Split(<tiktoken/Llama-3 pattern>, Isolated), ByteLevel(use_regex=False)] is supported")
        cfg["pretok"] = _lib.PRETOK_LLAMA3
    else:
        raise UnsupportedConfig(f"pre_tokenizer {pt['type']} is not on the accelerated path")
    if m["type"] == "BPE":
        cfg["model"] = _lib.MODEL_BPE
        for k in ("dropout", "unk_token", "continuing_subword_prefix", "end_of_word_suffix"):
            if m.get(k):
                raise UnsupportedConfig(f"BPE option {k} is not on the accelerated path")
        if m.get("byte_fallback") or m.get("fuse_unk"):
            raise UnsupportedConfig("BPE byte_fallback / fuse_unk are not on the accelerated path")
        cfg["ignore_merges"] = int(m.get("ignore_merges", False))
        cfg["merges"] = [tuple(x.split(" ")) if isinstance(x, str) else tuple(x) for x in m["merges"]]
    elif m["type"] == "WordPiece":
        cfg["model"] = _lib.MODEL_WORDPIECE
        cfg["unk"] = m["unk_token"]
        cfg["prefix"] = m["continuing_subword_prefix"]
        cfg["max_chars"] = m["max_input_chars_per_word"]
    else:
        raise UnsupportedConfig(f"model {m['type']} is not on the accelerated path")
    cfg["vocab"] = m["vocab"]
    cfg["added_tokens"] = list(js.get("added_tokens", []))
    if norm and cfg["model"] != _lib.MODEL_WORDPIECE:
        raise UnsupportedConfig("BertNormalizer is on the accelerated path in front of WordPiece only")
    if norm and any(t.get("content") and t.get("normalized", not t.get("special", False)) for t in cfg["added_tokens"]):
        # added_vocabulary.rs:545-560: such tokens are searched in the NORMALIZED text of every piece; only the special
        # (non-normalized) ones, which are cut out of the raw text before the normalizer runs, are mirrored
        raise UnsupportedConfig("added tokens with normalized=true behind a normalizer are not on the accelerated path")
    if template is not None and template["trim"] is not None and (cfg["model"] != _lib.MODEL_BPE or cfg["pretok"] == _lib.PRETOK_WHITESPACE):
        raise UnsupportedConfig("trim_offsets needs a byte-level BPE pipeline")
    cfg["template"] = template
    cfg["decoder"] = js.get("decoder")
    cfg["truncation"] = parse_truncation(js.get("truncation"))
    cfg["padding"] = parse_padding(js.get("padding"))
    return cfg


def decoder_spec(decoder, added_tokens):
    """tokenizer.json's decoder and the added vocabulary (objects with content, id, special, normalized) -> (b2t_decoder_spec,
    the arrays it points into), or (None, reason) for a decoder the device does not run"""
    ty = None if decoder is None else decoder.get("type")
    kinds = {None: _lib.DECODER_NONE, "ByteLevel": _lib.DECODER_BYTELEVEL, "WordPiece": _lib.DECODER_WORDPIECE}
    if ty not in kinds:
        return None, f"decoder {ty} is not supported on the device (ByteLevel, WordPiece and no decoder are)"
    toks = [t for t in added_tokens if t.content]
    tb, to = _pack([t.content for t in toks], np.uint32)
    ti = np.asarray([t.id for t in toks], dtype=np.uint32)
    tf = np.asarray([(_lib.ADDED_SPECIAL if t.special else 0) | (_lib.ADDED_NORMALIZED if t.normalized else 0) for t in toks], dtype=np.uint8)
    sp = _lib.DecoderSpec()
    sp.struct_size = ctypes.sizeof(_lib.DecoderSpec)
    sp.kind = kinds[ty]
    sp.prefix = decoder.get("prefix", "##").encode("utf-8") if ty == "WordPiece" else None
    sp.cleanup = int(bool(decoder.get("cleanup", True))) if ty == "WordPiece" else 0
    sp.n_added = len(toks)
    sp.added_bytes, sp.added_off, sp.added_ids, sp.added_flags = tb.ctypes.data, to.ctypes.data, ti.ctypes.data, tf.ctypes.data
    return sp, (tb, to, ti, tf)


def engine_config(cfg, device=-1):
    """parse_tokenizer_json's dict -> (b2t_config, the arrays it points into)"""
    vocab = cfg["vocab"]
    toks = list(vocab.keys())
    vb, vo = _pack(toks, np.uint32)
    vi = np.fromiter((vocab[t] for t in toks), dtype=np.uint32, count=len(toks))
    mb, mo = _pack([s for ab in cfg["merges"] for s in ab], np.uint32)
    c = _lib.Config()
    c.struct_size = ctypes.sizeof(_lib.Config)
    c.model, c.pretok = cfg["model"], cfg["pretok"]
    c.add_prefix_space, c.ignore_merges = cfg["add_prefix_space"], cfg["ignore_merges"]
    c.n_vocab, c.vocab_bytes, c.vocab_off, c.vocab_ids = len(toks), vb.ctypes.data, vo.ctypes.data, vi.ctypes.data
    c.n_merges, c.merge_bytes, c.merge_off = len(cfg["merges"]), mb.ctypes.data, mo.ctypes.data
    c.unk_token = cfg["unk"].encode("utf-8") if cfg["unk"] is not None else None
    c.continuing_subword_prefix = cfg["prefix"].encode("utf-8")
    c.max_input_chars_per_word = cfg["max_chars"]
    c.device = device
    c.bert_normalizer = cfg.get("normalizer", 0)
    return c, (vb, vo, vi, mb, mo)


NO_WORD = 0xFFFFFFFF  # word id of a token the post-processor added (the reference reports None)


class _ResultOwner:
    """Keeps a b2t_result (and the pinned buffers the zero-copy views point into) alive; frees it with the last view holder.
    It also keeps the Tokenizer whose engine made the result, since a result must be freed before its engine."""

    def __init__(self, res, tok):
        self._res, self._tok = res, tok

    def __del__(self):
        r, self._res = self._res, None
        if r:
            try:
                _lib.lib().b2t_result_free(r)
            except Exception:
                pass


class _Rows(tuple):
    """(ids, offsets or None, word ids or None, row_ptr) of one engine call.  `owner`: the _ResultOwner that keeps the
    arrays valid when they are zero-copy views, else None."""
    owner = None


class BatchEncoding:
    """The whole batch as a CSR (numpy arrays copied out of the engine's pinned buffers).  `type_ids`,
    `special_tokens_mask` and `attention_mask` are None unless a special-token template / padding was applied; tokens
    those added carry offsets (0, 0) and word id NO_WORD."""

    def __init__(self, ids, offsets, word_ids, row_ptr, type_ids=None, special_tokens_mask=None, attention_mask=None, sequence_ids=None):
        self.ids, self.offsets, self.word_ids, self.row_ptr = ids, offsets, word_ids, row_ptr
        self.type_ids, self.special_tokens_mask, self.attention_mask = type_ids, special_tokens_mask, attention_mask
        self.sequence_ids = sequence_ids  # int8, -1 = none (special / pad token); only set for pairs of sequences
        self.token_text = None            # {token index: str}: added tokens whose text is a wider span than their content (lstrip / rstrip)
        self._owner = None                # the _ResultOwner of the engine result that zero-copy arrays are views of

    def _remap_text(self, src, new_to_old):
        """carry src.token_text over to this CSR, whose token i is src's token new_to_old[i]"""
        if src.token_text:
            keys = np.fromiter(src.token_text, dtype=np.int64)
            slot = np.full(len(src.ids), -1, dtype=np.int64)
            slot[keys] = np.arange(len(keys))
            hit = np.flatnonzero(slot[new_to_old] >= 0)
            vals = list(src.token_text.values())
            self.token_text = {int(i): vals[int(slot[new_to_old[i]])] for i in hit}
        return self

    @property
    def n_tokens(self):
        return int(self.row_ptr[-1])


class Encoding:
    """One row of a BatchEncoding with the attribute names of `tokenizers.Encoding` (bindings/python/src/encoding.rs:
    133-225).  A view: the lists are made when an attribute is read, so a batch of millions of sequences costs nothing
    for the attributes nobody looks at."""
    __slots__ = ("_tok", "_be", "_a", "_b", "_pad_token", "overflowing")

    def __init__(self, tok, be, a, b):
        self._tok, self._be, self._a, self._b = tok, be, a, b  # tokens [a, b) of be
        self._pad_token, self.overflowing = None, ()           # overflowing: parts cut off by truncation (a list then)

    def __len__(self):
        return self._b - self._a

    def _col(self, arr):
        return None if arr is None else arr[self._a:self._b]

    @property
    def ids(self):
        return self._be.ids[self._a:self._b].tolist()

    @property
    def offsets(self):
        if self._be.offsets is None:  # encode_batch_fast (OffsetType::None): the reference reports (0, 0) everywhere
            return [(0, 0)] * len(self)
        return [tuple(x) for x in self._be.offsets[self._a:self._b].tolist()]

    @property
    def word_ids(self):
        if self._be.word_ids is None:  # encode_batch_fast: no word indices either
            return [None] * len(self)
        return [None if w == NO_WORD else w for w in self._be.word_ids[self._a:self._b].tolist()]

    words = word_ids

    @property
    def tokens(self):
        ids, attn, text = self.ids, self._col(self._be.attention_mask), self._be.token_text
        out = [self._tok.id_to_token(i) for i in ids]
        if attn is not None:
            out = [t if m else self._pad_token for t, m in zip(out, attn.tolist())]
        if text:
            for k in range(len(out)):
                if self._a + k in text:
                    out[k] = text[self._a + k]
        return out

    @property
    def type_ids(self):
        t = self._col(self._be.type_ids)
        return [0] * len(self) if t is None else t.tolist()

    @property
    def attention_mask(self):
        m = self._col(self._be.attention_mask)
        return [1] * len(self) if m is None else m.tolist()

    @property
    def special_tokens_mask(self):
        m = self._col(self._be.special_tokens_mask)
        return [0] * len(self) if m is None else m.tolist()

    @property
    def sequence_ids(self):
        """Known differences from the reference (host-side bookkeeping outside the accelerated path, found by differential runs
        against tokenizers 0.22.2): the reference derives this list from `sequence_ranges`, which it clears on truncation and
        does not set for pre-tokenized input -- padded pre-tokenized encodings report 0 for their pad tokens there (None here),
        and the tokens of the second sequence of a pair that was truncated into overflowing parts report None there (1 here).
        ids, offsets, word_ids, type_ids, masks, tokens and overflowing are identical."""
        q = self._col(self._be.sequence_ids)
        if q is not None:
            return [None if v < 0 else v for v in q.tolist()]
        m = self._col(self._be.special_tokens_mask)
        return [0] * len(self) if m is None else [None if sp else 0 for sp in m.tolist()]

    @property
    def n_sequences(self):
        q = self._col(self._be.sequence_ids)
        return 1 if q is None or q.size == 0 else max(int(q.max()) + 1, 1)

    def _pad(self, target, pad_id, pad_type_id, pad_token, left):
        """Encoding::pad (tokenizer/encoding.rs:465-560): this row gets arrays of its own"""
        for o in self.overflowing:
            o._pad(target, pad_id, pad_type_id, pad_token, left)
        n = len(self)
        k = target - n
        if k <= 0:
            return
        be = self._be
        cat = (lambda pad, x: np.concatenate([pad, x])) if left else (lambda pad, x: np.concatenate([x, pad]))
        col = lambda arr, default: default if arr is None else arr[self._a:self._b]
        self._be = BatchEncoding(
            cat(np.full(k, pad_id, dtype=np.uint32), col(be.ids, None)),
            None if be.offsets is None else cat(np.zeros((k, 2), dtype=np.uint32), col(be.offsets, None)),
            None if be.word_ids is None else cat(np.full(k, NO_WORD, dtype=np.uint32), col(be.word_ids, None)),
            np.array([0, target], dtype=np.uint64),
            cat(np.full(k, pad_type_id, dtype=np.uint32), col(be.type_ids, np.zeros(n, dtype=np.uint32))),
            cat(np.ones(k, dtype=np.uint8), col(be.special_tokens_mask, np.zeros(n, dtype=np.uint8))),
            cat(np.zeros(k, dtype=np.uint8), col(be.attention_mask, np.ones(n, dtype=np.uint8))),
            None if be.sequence_ids is None else cat(np.full(k, -1, dtype=np.int8), col(be.sequence_ids, None)))
        if be.token_text:
            shift = (k if left else 0) - self._a
            self._be.token_text = {i + shift: t for i, t in be.token_text.items() if self._a <= i < self._b}
        self._a, self._b, self._pad_token = 0, target, pad_token

    def __repr__(self):
        return f"Encoding(num_tokens={len(self)}, attributes=[ids, type_ids, tokens, offsets, attention_mask, special_tokens_mask, overflowing])"


def special_token_count(template, is_pair):
    """PostProcessor::added_tokens (template.rs:647-653, bert.rs, roberta.rs): the special tokens the template adds to a
    single sequence or a pair (0 without a template, or for a pair without a pair template)"""
    pieces = None if template is None else template["pair" if is_pair else "single"]
    return sum(1 for p in pieces or () if p[0] == "special")


def truncation_budget(truncation, template, is_pair, add_special_tokens):
    """TokenizerImpl::post_process step 1 (tokenizer/mod.rs:1265-1317): truncation's max_length less the special tokens
    the post-processor will add"""
    n_added = special_token_count(template, is_pair) if add_special_tokens else 0
    if truncation["max_length"] < n_added:
        raise ValueError("truncation max_length is smaller than the number of special tokens the post-processor adds")
    return truncation["max_length"] - n_added


def truncation_spans(n, max_len, stride, direction):
    """Encoding::truncate (tokenizer/encoding.rs:307-388) on a sequence of n tokens -> [(a, b)]: the kept part first, then
    the overflowing parts (each max_len long, consecutive ones sharing `stride` tokens)"""
    if n <= max_len:
        return [(0, n)]
    if max_len == 0:
        return [(0, 0), (0, n)]  # an empty kept part, the whole sequence overflows (encoding.rs:313-317)
    if stride >= max_len:
        raise ValueError(f"`stride` must be strictly less than `max_len={max_len}` (the maximum length minus the special tokens)")
    step, spans = max_len - stride, []
    if direction == "right":
        for a in range(0, n, step):
            b = min(a + max_len, n)
            spans.append((a, b))
            if b == n:
                break
    else:
        for stop in range(n, 0, -step):
            a = max(stop - max_len, 0)
            spans.append((a, stop))
            if a == 0:
                break
    return spans


def trim_spans(offsets, ld, tr, first, add_prefix_space):
    """ByteLevel::process_offsets (pre_tokenizers/byte_level.rs:202-234): offsets [T, 2] shrink by the token's leading /
    trailing space characters ld / tr, except that with add_prefix_space a first token of a sequence (`first`), or one
    at offset 0, keeps a single leading space.  -> uint32 [T, 2]"""
    ld, tr = np.asarray(ld, dtype=np.int64), np.asarray(tr, dtype=np.int64)
    o = np.asarray(offsets, dtype=np.int64).reshape(-1, 2)
    o0, o1 = o[:, 0], o[:, 1]
    keep = (first | (o0 == 0)) & bool(add_prefix_space) & (ld == 1)
    n0 = np.where((ld > 0) & ~keep, np.minimum(o0 + ld, o1), o0)
    n1 = np.where((tr > 0) & (o1 >= tr), np.maximum(o1 - tr, n0), o1)
    return np.stack([n0, n1], axis=1).astype(np.uint32)


def trim_offsets(be, ld, tr, add_prefix_space):
    """trim_spans on the whole CSR.  ld / tr: per token, the number of leading / trailing space characters of its text."""
    if be.offsets is None or be.ids.size == 0:
        return be
    first = np.zeros(be.ids.size, dtype=bool)
    first[be.row_ptr[:-1][np.diff(be.row_ptr) > 0].astype(np.int64)] = True
    out = BatchEncoding(be.ids, trim_spans(be.offsets, ld, tr, first, add_prefix_space), be.word_ids, be.row_ptr, be.type_ids,
                        be.special_tokens_mask)
    out.token_text = be.token_text
    return out


def truncate_csr(be, extra, max_length, stride, direction):
    """truncation_spans for every sequence of the CSR: a sequence longer than max_length becomes several rows, the kept
    part first, then its overflowing parts.  extra: per-token arrays cut the same way.
    -> (BatchEncoding of all parts, extra arrays, part_doc int64[parts] = document of each part)"""
    seg_a, seg_b, seg_doc = [], [], []
    rows = be.row_ptr.astype(np.int64).tolist()
    for d, (s, e) in enumerate(zip(rows[:-1], rows[1:])):
        for a, b in truncation_spans(e - s, max_length, stride, direction):
            seg_a.append(s + a); seg_b.append(s + b); seg_doc.append(d)
    seg_a, seg_b = np.asarray(seg_a, dtype=np.int64), np.asarray(seg_b, dtype=np.int64)
    lens = seg_b - seg_a
    rp = np.zeros(len(lens) + 1, dtype=np.uint64)
    np.cumsum(lens, out=rp[1:])
    idx = np.repeat(seg_a - rp[:-1].astype(np.int64), lens) + np.arange(int(rp[-1]), dtype=np.int64)
    take = lambda x: None if x is None else x[idx]
    return (BatchEncoding(be.ids[idx], take(be.offsets), take(be.word_ids), rp)._remap_text(be, idx), [take(x) for x in extra],
            np.asarray(seg_doc, dtype=np.int64))


def post_process(be, template):
    """TokenizerImpl::post_process for single sequences (tokenizer/mod.rs:1265-1317 -> processors/template.rs
    `apply_template`): the template's special tokens go in front of / behind every sequence of the CSR."""
    pre, post = template["pre"], template["post"]
    n = len(be.row_ptr) - 1
    counts = np.diff(be.row_ptr).astype(np.int64)
    T, extra = int(counts.sum()), len(pre) + len(post)
    new_rp = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(counts + extra, out=new_rp[1:])
    NT = int(new_rp[-1])
    pos = np.arange(T, dtype=np.int64) + np.repeat(np.arange(n, dtype=np.int64) * extra + len(pre), counts)
    ids = np.zeros(NT, dtype=np.uint32); ids[pos] = be.ids
    type_ids = np.zeros(NT, dtype=np.uint32); type_ids[pos] = template["type_id"]
    special = np.ones(NT, dtype=np.uint8); special[pos] = 0
    offs = wid = None
    if be.offsets is not None:
        offs = np.zeros((NT, 2), dtype=np.uint32); offs[pos] = be.offsets
    if be.word_ids is not None:
        wid = np.full(NT, NO_WORD, dtype=np.uint32); wid[pos] = be.word_ids
    starts, ends = new_rp[:-1].astype(np.int64), new_rp[1:].astype(np.int64)
    for j, (tid, ty) in enumerate(pre):
        ids[starts + j] = tid; type_ids[starts + j] = ty
    for j, (tid, ty) in enumerate(post):
        ids[ends - len(post) + j] = tid; type_ids[ends - len(post) + j] = ty
    out = BatchEncoding(ids, offs, wid, new_rp, type_ids, special)
    if be.token_text:
        out.token_text = {int(pos[i]): t for i, t in be.token_text.items()}
    return out


_CHAR_BYTES = None


def _char_bytes():
    """inverse of the byte-level alphabet (pre_tokenizers/byte_level.rs:15-39): character -> byte"""
    global _CHAR_BYTES
    if _CHAR_BYTES is None:
        keep = list(range(0x21, 0x7F)) + list(range(0xA1, 0xAD)) + list(range(0xAE, 0x100))
        cs, n = {b: chr(b) for b in keep}, 0
        for b in range(256):
            if b not in cs:
                cs[b] = chr(256 + n); n += 1
        _CHAR_BYTES = {c: b for b, c in cs.items()}
    return _CHAR_BYTES


def _view(ptr, count, dtype):
    if not ptr or count == 0:
        return np.zeros(0, dtype=dtype)
    nbytes = count * np.dtype(dtype).itemsize
    return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint8)), shape=(nbytes,)).view(dtype)


def _read_result(tok, res, views, zero_copy=False):
    """A b2t_result of tok's engine -> (numpy arrays, owner).  views(L, res) returns views of the result's pinned host
    buffers (None for an array that was not asked for).  Without zero_copy the arrays are copies, the result is freed
    and owner is None; with it they are the views themselves and owner is the _ResultOwner that frees the result:
    whoever keeps the views must keep the owner."""
    L = _lib.lib()
    if zero_copy:
        owner = _ResultOwner(res, tok)
        return views(L, res), owner
    try:
        return tuple(None if a is None else a.copy() for a in views(L, res)), None
    finally:
        L.b2t_result_free(res)


def _device_view(torch, ptr, count, dtype, device):
    """a torch tensor over `count` elements of device memory the engine owns (no copy)"""
    typestr = {torch.uint8: "|u1", torch.int32: "<i4", torch.int64: "<i8"}[dtype]

    class _Mem:
        __cuda_array_interface__ = {"shape": (count,), "typestr": typestr, "data": (ptr, False), "version": 2}
    return torch.as_tensor(_Mem(), device=device)


def _byte_span(data, a0, b0, o0, o1, byte_offsets):
    """the byte span in data of a token with offsets (o0, o1) in the document data[a0:b0]; char offsets count the
    document's UTF-8 lead bytes"""
    if byte_offsets:
        return a0 + o0, a0 + o1
    lead = np.flatnonzero((data[a0:b0] & 0xC0) != 0x80)
    at = lambda o: a0 + int(lead[o]) if o < lead.size else b0
    return at(o0), at(o1)


class Tokenizer:
    def __init__(self, tokenizer_json, device=-1):
        js = json.loads(tokenizer_json) if isinstance(tokenizer_json, (str, bytes)) else tokenizer_json
        self._init_host(parse_tokenizer_json(js))
        self._create_engine(device)

    def _init_host(self, cfg):
        self._cfg = cfg
        self._vocab = cfg["vocab"]
        self._vocab_r = None
        self._template = cfg["template"]
        self._truncation, self._padding = cfg["truncation"], cfg["padding"]
        self._decoder = cfg["decoder"]
        self._trim = None
        self._added = None
        self._dev_added, self._added_strip = False, False
        if any(t.get("content") for t in cfg["added_tokens"]):
            self._added = added.AddedVocabulary(cfg["added_tokens"], self._rust_class_table())

    @staticmethod
    def _rust_class_table():
        """Rust-regex \\w / \\s classes per code point from the library's own tables (a host-only call, no GPU work)."""
        tbl = np.zeros(0x110000, dtype=np.uint8)
        _lib.check(_lib.lib().b2t_unicode_class_table(1, tbl.ctypes.data))
        return tbl

    def _create_engine(self, device):
        L = _lib.lib()
        c, _keep = engine_config(self._cfg, device)
        self._device = device
        h = ctypes.c_void_p()
        rc = L.b2t_engine_create(ctypes.byref(c), ctypes.byref(h))
        if rc == _lib.B2T_ERR_UNSUPPORTED:
            raise UnsupportedConfig(L.b2t_last_error().decode())
        _lib.check(rc)
        self._h = h
        self._register_added()

    def _register_added(self):
        """Hand the added vocabulary to the engine: to the extraction (b2t_engine_set_added_tokens) and, with the id -> string
        map it changes, to the decoder (b2t_engine_set_decoder)."""
        self._register_added_tokens()
        self._set_decoder()

    def _set_decoder(self):
        """b2t_engine_set_decoder; a refusal only makes the device decode entry points unavailable (its reason is kept
        for them to raise), it never fails construction"""
        self._decoder_refused = "the tokenizer has no engine"
        if getattr(self, "_h", None) is None:
            return
        L = _lib.lib()
        sp, keep = decoder_spec(self._decoder, [] if self._added is None else list(self._added.tokens.values()))
        if sp is None:
            L.b2t_engine_set_decoder(self._h, None)
            self._decoder_refused = keep
            return
        rc = L.b2t_engine_set_decoder(self._h, ctypes.byref(sp))
        self._decoder_refused = None if rc == _lib.B2T_OK else L.b2t_last_error().decode("utf-8", "replace")

    def _register_added_tokens(self):
        """Hand the added vocabulary to the engine (b2t_engine_set_added_tokens): the extraction then runs on the device.
        Configurations the device path refuses (add_prefix_space) keep the host extraction of added.py in front of the engine."""
        self._dev_added = False
        if getattr(self, "_h", None) is None:
            return
        L = _lib.lib()
        toks = [] if self._added is None else list(self._added.by_content.values())
        if not toks:
            L.b2t_engine_set_added_tokens(self._h, 0, None, None, None, None)
            return
        tb, to = _pack([t.content for t in toks], np.uint32)
        ti = np.asarray([t.id for t in toks], dtype=np.uint32)
        tf = np.asarray([(_lib.ADDED_SINGLE_WORD if t.single_word else 0) | (_lib.ADDED_LSTRIP if t.lstrip else 0) |
                         (_lib.ADDED_RSTRIP if t.rstrip else 0) | (_lib.ADDED_NORMALIZED if t.normalized else 0) for t in toks], dtype=np.uint8)
        rc = L.b2t_engine_set_added_tokens(self._h, len(toks), tb.ctypes.data, to.ctypes.data, ti.ctypes.data, tf.ctypes.data)
        if rc == _lib.B2T_ERR_UNSUPPORTED:
            return
        _lib.check(rc)
        self._dev_added = True
        self._added_strip = any(t.lstrip or t.rstrip for t in toks)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            _lib.lib().b2t_engine_destroy(h)
            self._h = None

    # ---- construction (tokenizer/mod.rs:468-476)
    @staticmethod
    def from_str(s, device=-1):
        return Tokenizer(s, device)

    @staticmethod
    def from_file(path, device=-1):
        import gzip
        opener = gzip.open if str(path).endswith(".gz") else open
        with opener(path, "rb") as f:
            return Tokenizer(f.read().decode("utf-8"), device)

    # ---- vocabulary helpers (added tokens shadow the model's vocabulary: added_vocabulary.rs:205-238)
    def get_vocab_size(self, with_added_tokens=True):
        n = len(self._vocab)
        if with_added_tokens and self._added is not None:
            n += sum(1 for t in self._added.tokens.values() if self._vocab.get(t.content) != t.id)
        return n

    def get_vocab(self, with_added_tokens=True):
        v = dict(self._vocab)
        if with_added_tokens and self._added is not None:
            v.update({t.content: t.id for t in self._added.tokens.values()})
        return v

    def num_special_tokens_to_add(self, is_pair):
        return special_token_count(self._template, is_pair)

    def _add(self, tokens, special):
        """AddedVocabulary::add_tokens (added_vocabulary.rs:270-340): a token keeps the model's id when its content is in the
        vocabulary, otherwise it gets the next free id; returns how many were new"""
        entries = [] if self._added is None else [
            {"id": t.id, "content": t.content, "single_word": t.single_word, "lstrip": t.lstrip, "rstrip": t.rstrip,
             "normalized": t.normalized, "special": t.special} for t in self._added.tokens.values()]
        known = {e["content"]: e for e in entries}
        # added_vocabulary.rs add_tokens: a new token gets max(id of the added tokens) + 1 when that lies beyond the model's
        # vocabulary, else the model's vocabulary size (NOT its largest id + 1: the two differ for vocabularies with gaps)
        vocab_size, max_added = len(self._vocab), max([e["id"] for e in entries] + [-1])
        nxt = max_added + 1 if max_added >= vocab_size else vocab_size
        added_n = 0
        for t in tokens:
            d = {"content": t} if isinstance(t, str) else {k: getattr(t, k) for k in ("content", "single_word", "lstrip", "rstrip", "normalized") if hasattr(t, k)}
            if not d.get("content"):
                continue
            d.setdefault("single_word", False); d.setdefault("lstrip", False); d.setdefault("rstrip", False)
            d["special"] = special
            if isinstance(t, str) or "normalized" not in d:
                d["normalized"] = not special
            old = known.get(d["content"])
            if old is not None and all(old[k] == d[k] for k in ("single_word", "lstrip", "rstrip", "normalized", "special")):
                continue
            if d["content"] in self._vocab:
                d["id"] = self._vocab[d["content"]]
            elif old is not None:
                d["id"] = old["id"]
            else:
                d["id"], nxt = nxt, nxt + 1
            if old is not None:
                entries.remove(old)
            entries.append(d); known[d["content"]] = d
            added_n += 1
        self._added = added.AddedVocabulary(entries, self._rust_class_table()) if entries else None
        self._trim = None
        self._register_added()
        return added_n

    def add_tokens(self, tokens):
        return self._add(tokens, False)

    def add_special_tokens(self, tokens):
        return self._add(tokens, True)

    def token_to_id(self, token):
        if self._added is not None and token in self._added.by_content:
            return self._added.by_content[token].id
        return self._vocab.get(token)

    def id_to_token(self, i):
        if self._added is not None and int(i) in self._added.tokens:
            return self._added.tokens[int(i)].content
        if self._vocab_r is None:
            self._vocab_r = {v: k for k, v in self._vocab.items()}
        return self._vocab_r.get(int(i))

    @property
    def handle(self):
        return self._h

    # ---- encode
    def _engine_rows(self, data, row_off, flags, zero_copy=False):
        """The C-ABI call: packed rows in host memory -> _Rows (ids, offsets or None, word ids or None, row_ptr): copies,
        or with zero_copy views of the result whose _ResultOwner is the _Rows' `owner`."""
        n_rows = len(row_off) - 1
        L = _lib.lib()
        res = ctypes.c_void_p()
        _lib.check(L.b2t_encode_batch(self._h, data.ctypes.data if data.size else None, row_off.ctypes.data, n_rows, flags, ctypes.byref(res)))

        def views(L, res):
            T = L.b2t_result_n_tokens(res)
            return (_view(L.b2t_result_ids(res), T, np.uint32),
                    _view(L.b2t_result_offsets(res), 2 * T, np.uint32).reshape(-1, 2) if flags & _lib.WANT_OFFSETS else None,
                    _view(L.b2t_result_word_ids(res), T, np.uint32) if flags & _lib.WANT_WORD_IDS else None,
                    _view(L.b2t_result_row_ptr(res), n_rows + 1, np.uint64))
        arrays, owner = _read_result(self, res, views, zero_copy)
        rows = _Rows(arrays)
        rows.owner = owner
        return rows

    # ---- truncation / padding (bindings/python/src/tokenizer.rs:700-820)
    def enable_truncation(self, max_length, stride=0, strategy="longest_first", direction="right"):
        if strategy not in ("longest_first", "only_first", "only_second") or direction not in ("left", "right"):
            raise ValueError("unknown truncation strategy / direction")
        self._truncation = {"max_length": int(max_length), "stride": int(stride), "strategy": strategy, "direction": direction}

    def no_truncation(self):
        self._truncation = None

    @property
    def truncation(self):
        return None if self._truncation is None else dict(self._truncation)

    def enable_padding(self, direction="right", pad_id=0, pad_type_id=0, pad_token="[PAD]", length=None, pad_to_multiple_of=None):
        if direction not in ("left", "right"):
            raise ValueError("unknown padding direction")
        self._padding = {"length": length, "direction": direction, "pad_to_multiple_of": pad_to_multiple_of, "pad_id": int(pad_id),
                         "pad_type_id": int(pad_type_id), "pad_token": pad_token}

    def no_padding(self):
        self._padding = None

    @property
    def padding(self):
        return None if self._padding is None else dict(self._padding)

    def _encode_core(self, data, doc_off, flags, extract_added_tokens, zero_copy=False):
        """added-token extraction -> engine -> stitching.  -> (BatchEncoding of the plain sequences, trim counts or None);
        with zero_copy the BatchEncoding's arrays may be views of the engine's result, kept valid by its `_owner`"""
        if extract_added_tokens and self._dev_added:
            try:
                return self._encode_device_extraction(data, doc_off, flags, zero_copy)
            except _lib.B2TError as ex:
                if ex.code != _lib.B2T_ERR_UNSUPPORTED:
                    raise  # (spans outside the device limits: split on the host instead)
        return self._encode_host_extraction(data, doc_off, flags, extract_added_tokens, zero_copy)

    def _encode_device_extraction(self, data, doc_off, flags, zero_copy):
        """The extraction runs on the device; added tokens come back marked (bit 31 of the id).  Their matched spans are
        read off the offsets where the host needs the text (lstrip / rstrip tokens, offset trimming)."""
        tp = self._template
        need_text = self._added_strip or (tp is not None and tp["trim"] is not None and bool(flags & _lib.WANT_OFFSETS))
        fl = flags | _lib.FLAG_ADDED_IDS | (_lib.WANT_OFFSETS if need_text else 0)
        rows = self._engine_rows(data, doc_off, fl, zero_copy)
        ids, offs, wid, rp = rows
        marked = np.flatnonzero(ids >> 31)
        ids &= np.uint32(0x7FFFFFFF)
        added_at = []
        if need_text and marked.size:
            docs_of = np.searchsorted(rp, marked, side="right") - 1
            for i, d in zip(marked.tolist(), docs_of.tolist()):
                added_at.append((i, *_byte_span(data, int(doc_off[d]), int(doc_off[d + 1]), int(offs[i, 0]), int(offs[i, 1]),
                                                 bool(flags & _lib.OFFSETS_BYTES))))
        return self._plain_encoding(data, ids, offs if flags & _lib.WANT_OFFSETS else None, wid, rp, added_at, rows)

    def _encode_host_extraction(self, data, doc_off, flags, extract_added_tokens, zero_copy):
        """added.py cuts the documents at the added tokens, the engine encodes the pieces, and the rows are stitched back."""
        row_off, parts, cut, added_at = doc_off, None, False, []
        if extract_added_tokens and self._added is not None:
            row_off, parts, cut = added.split_batch(self._added, data, doc_off)
        rows = self._engine_rows(data, row_off, flags | (_lib.NO_ADDED_TOKENS if self._added is not None else 0), zero_copy)
        ids, offs, wid, rp = rows
        if cut:
            ids, offs, wid, rp, added_at = added.stitch_rows(data, doc_off, parts, ids, offs, wid, rp, bool(flags & _lib.OFFSETS_BYTES))
        return self._plain_encoding(data, ids, offs, wid, rp, added_at, rows)

    def _plain_encoding(self, data, ids, offs, wid, rp, added_at, rows):
        """-> (BatchEncoding, trim counts or None).  added_at: (token index, byte span in data) of the added tokens whose
        matched text the host needs; rows: what _engine_rows returned, whose owner the BatchEncoding keeps."""
        tp = self._template
        trim = None
        if tp is not None and tp["trim"] is not None and offs is not None:
            lead, trail = self._trim_tables()
            ld, tr = lead[ids], trail[ids]
            for i, a, b in added_at:
                ld[i], tr[i] = self._span_spaces(data, a, b)
            trim = (ld, tr)
        be = BatchEncoding(ids, offs, wid, rp)
        be._owner = getattr(rows, "owner", None)   # (a replacement of the engine seam may return a plain tuple)
        for i, a, b in added_at:  # Token::new(id, value = the matched span): differs from the content after lstrip / rstrip
            tok = self._added.tokens[int(ids[i])]
            if b - a != len(tok.content.encode("utf-8")):
                if be.token_text is None:
                    be.token_text = {}
                be.token_text[i] = bytes(data[a:b]).decode("utf-8", "replace")
        return be, trim

    def _finish(self, be, trim, add_special_tokens):
        """the post-processor: offset trimming, then the special-token template"""
        tp = self._template
        if trim is not None:
            be = trim_offsets(be, trim[0], trim[1], tp["trim"])
        if add_special_tokens and tp is not None and (tp["pre"] or tp["post"]):
            be = post_process(be, tp)
        return be

    def encode_batch_csr(self, data, doc_off, offsets=True, word_ids=True, byte_offsets=False, add_special_tokens=False,
                         extract_added_tokens=True, zero_copy=False):
        """Packed batch in (np.uint8[N], np.uint64[n+1]) -> BatchEncoding.  Host buffers; copies happen inside.

        extract_added_tokens: run the reference's added-token extraction (added_vocabulary.rs:523-564) on the host before
        the engine when the tokenizer has added tokens -- a byte search over the whole buffer; pass False when the
        caller knows the text holds none (then this is exactly one b2t_encode_batch call).
        add_special_tokens: apply the post-processor's single-sequence template (default False here: the CSR entry
        point is the raw hot path; `encode_batch` follows the reference's default of True).
        Truncation / padding settings change the shape of the result (overflowing parts, pad tokens) and are honoured
        by `encode_batch` / `encode`, not here."""
        if self._truncation is not None or self._padding is not None:
            raise UnsupportedConfig("truncation / padding are enabled: use encode_batch (the CSR entry point returns plain sequences)")
        data = np.ascontiguousarray(data, dtype=np.uint8)
        doc_off = np.ascontiguousarray(doc_off, dtype=np.uint64)
        flags = (_lib.WANT_OFFSETS if offsets else 0) | (_lib.WANT_WORD_IDS if word_ids else 0) | (_lib.OFFSETS_BYTES if byte_offsets else 0)
        be, trim = self._encode_core(data, doc_off, flags, extract_added_tokens, bool(zero_copy))
        out = self._finish(be, trim, add_special_tokens)
        out._owner = be._owner   # the views die with the BatchEncoding
        return out

    # ---- dense mode: template + truncation + padding on the device (include/b2t.h b2t_encode_batch_dense, b2t_encode_pairs_dense)
    def _dense_fields(self, sp, want_mask, overflow=False, offsets=False, trim_offsets=False, special_mask=False, sequence_ids=False,
                      word_ids=False):
        """the padding / truncation fields b2t_dense_spec and b2t_pair_dense_spec share, filled into sp; overflow / offsets:
        return_overflowing_tokens / return_offsets_mapping; trim_offsets: offset rows as the post-processor leaves them
        (trimmed where it trims); special_mask / sequence_ids / word_ids: the row metadata"""
        tr, pd = self._truncation, self._padding
        if pd is None:
            raise UnsupportedConfig("dense output needs padding enabled (enable_padding): rows must share one length")
        sp.struct_size = ctypes.sizeof(type(sp))
        sp.length = 0 if pd["length"] is None else int(pd["length"])
        sp.pad_to_multiple_of = int(pd["pad_to_multiple_of"] or 0)
        sp.max_length = 0 if tr is None else int(tr["max_length"])
        if tr is not None and sp.max_length == 0:
            raise UnsupportedConfig("truncation to max_length 0 has no dense form")
        sp.pad_id = pd["pad_id"]
        sp.truncate_left = int(tr is not None and tr["direction"] == "left")
        sp.pad_left = int(pd["direction"] == "left")
        sp.want_mask = int(want_mask)
        trims = self._template is not None and self._template["trim"] is not None
        if offsets and trims and not trim_offsets:
            raise UnsupportedConfig("offsets behind a post-processor that trims them (trim_offsets) have no dense form without trim_offsets=True")
        sp.stride = int(tr["stride"]) if (overflow and tr is not None) else 0
        sp.dense_flags = (_lib.DENSE_OVERFLOW if overflow else 0) | (_lib.DENSE_OFFSETS if offsets else 0)
        if offsets and trims:
            sp.dense_flags |= _lib.DENSE_TRIM_OFFSETS | (_lib.DENSE_TRIM_PREFIX_SPACE if self._template["trim"] else 0)
        if sequence_ids and self._template is None:
            # without a post-processor the reference's default_process keeps sequence ranges on the kept parts only, and a
            # sequence without ranges reads as sequence 0 over its whole length, padding included
            raise UnsupportedConfig("sequence ids of a tokenizer without a post-processor have no dense form")
        sp.dense_flags |= ((_lib.DENSE_SPECIAL_MASK if special_mask else 0) | (_lib.DENSE_SEQUENCE_IDS if sequence_ids else 0) |
                           (_lib.DENSE_WORD_IDS if word_ids else 0))
        return sp

    def dense_spec(self, add_special_tokens=True, want_mask=True, return_overflowing_tokens=False, return_offsets_mapping=False,
                   trim_offsets=False, return_special_tokens_mask=False, return_sequence_ids=False, return_word_ids=False):
        """The tokenizer's truncation / padding / single-sequence template as a b2t_dense_spec (+ the arrays it points to)."""
        tp = self._template
        pre = [t for t, _ in tp["pre"]] if (tp is not None and add_special_tokens) else []
        post = [t for t, _ in tp["post"]] if (tp is not None and add_special_tokens) else []
        sp = self._dense_fields(_lib.DenseSpec(), want_mask, return_overflowing_tokens, return_offsets_mapping, trim_offsets,
                                return_special_tokens_mask, return_sequence_ids, return_word_ids)
        keep = (np.asarray(pre, dtype=np.uint32), np.asarray(post, dtype=np.uint32))
        sp.n_pre, sp.n_post = len(pre), len(post)
        sp.pre_ids, sp.post_ids = (keep[0].ctypes.data if pre else None), (keep[1].ctypes.data if post else None)
        return sp, keep

    def pair_dense_spec(self, add_special_tokens=True, want_mask=True, return_overflowing_tokens=False, return_offsets_mapping=False,
                        trim_offsets=False, return_special_tokens_mask=False, return_sequence_ids=False, return_word_ids=False):
        """The tokenizer's truncation / padding / pair template as a b2t_pair_dense_spec (+ the arrays it points to).  The
        pieces come from the template's pair form (default_process without a post-processor: A type 0, B type 1); without
        special tokens the two sequence pieces stay, in their order and with their type ids (processors/template.rs:554-560).
        Overflowing parts keep the type id of their sequence (A 0, B 1), or the one the post-processor rewrites them to."""
        tp, tr, pd = self._template, self._truncation, self._padding
        pieces = [("seq", 0, 0), ("seq", 1, 1)] if tp is None else tp["pair"]
        if pieces is None:
            raise ValueError("the post-processor has no template for pairs of sequences")
        sp = self._dense_fields(_lib.PairDenseSpec(), want_mask, return_overflowing_tokens, return_offsets_mapping, trim_offsets,
                                return_special_tokens_mask, return_sequence_ids, return_word_ids)
        pieces = [p for p in pieces if p[0] == "seq" or add_special_tokens]
        ot = tp.get("overflow_type") if (tp is not None and add_special_tokens) else None   # (pairs.post_process's rule)
        sp.overflow_type_a, sp.overflow_type_b = (0, 1) if ot is None else (ot, ot)
        if tr is not None:
            if tr["stride"] and not return_overflowing_tokens:
                raise UnsupportedConfig("stride only shapes overflowing parts, which have no dense form")
            # the engine truncates the pair to max_length less the special tokens it is given: the budget of the reference
            sp.max_length = truncation_budget(tr, tp, True, add_special_tokens) + sum(1 for p in pieces if p[0] == "special")
            sp.strategy = {"longest_first": _lib.TRUNC_LONGEST_FIRST, "only_first": _lib.TRUNC_ONLY_FIRST, "only_second": _lib.TRUNC_ONLY_SECOND}[tr["strategy"]]
        sp.pad_type_id = pd["pad_type_id"]
        keep = (np.asarray([v if k == "special" else (_lib.PIECE_A if v == 0 else _lib.PIECE_B) for k, v, _ in pieces], dtype=np.uint32),
                np.asarray([t for _, _, t in pieces], dtype=np.uint32))
        sp.n_pieces, sp.piece_ids, sp.piece_types = len(pieces), keep[0].ctypes.data, keep[1].ctypes.data
        return sp, keep

    # The outputs of a dense call in the order of its dict: key, accessor, dtype, what a row holds ("pos": a value per
    # position, "pos2": a pair per position, "row": one value) and whether the spec asks for it.
    _DENSE_OUTPUTS = (
        ("input_ids", "b2t_result_dense_ids", np.uint32, "pos", lambda sp: True),
        ("token_type_ids", "b2t_result_type_ids", np.uint8, "pos", lambda sp: isinstance(sp, _lib.PairDenseSpec)),
        ("attention_mask", "b2t_result_attention_mask", np.uint8, "pos", lambda sp: sp.want_mask),
        ("lengths", "b2t_result_row_lengths", np.uint32, "row", lambda sp: True),
        ("overflow_to_sample_mapping", "b2t_result_row_sample", np.uint32, "row", lambda sp: sp.dense_flags & _lib.DENSE_OVERFLOW),
        ("offset_mapping", "b2t_result_dense_offsets", np.uint32, "pos2", lambda sp: sp.dense_flags & _lib.DENSE_OFFSETS),
        ("special_tokens_mask", "b2t_result_special_tokens_mask", np.uint8, "pos", lambda sp: sp.dense_flags & _lib.DENSE_SPECIAL_MASK),
        ("sequence_ids", "b2t_result_sequence_ids", np.int8, "pos", lambda sp: sp.dense_flags & _lib.DENSE_SEQUENCE_IDS),
        ("word_ids", "b2t_result_dense_word_ids", np.int32, "pos", lambda sp: sp.dense_flags & _lib.DENSE_WORD_IDS),   # -1 = None
    )

    def _dense_call(self, entry, data, doc_off, n_rows, sp):
        """b2t_encode_batch_dense / b2t_encode_pairs_dense -> {key: rows} of the outputs sp asks for, and "attention_mask":
        None without a mask; [R, L] per position ([R, L, 2] offsets) or [R] per row, R = n_rows without overflowing parts"""
        if self._added is not None and not self._dev_added and added.split_batch(self._added, data, doc_off)[2]:
            raise UnsupportedConfig("the batch contains added tokens and this configuration extracts them on the host: use encode_batch")
        L = _lib.lib()
        res = ctypes.c_void_p()
        _lib.check(getattr(L, entry)(self._h, data.ctypes.data if data.size else None, doc_off.ctypes.data, n_rows, ctypes.byref(sp), ctypes.byref(res)))
        asked = [want(sp) for *_, want in self._DENSE_OUTPUTS]

        def views(L, res):
            W, R = L.b2t_result_dense_length(res), L.b2t_result_dense_rows(res)
            shapes = {"pos": (R, W), "pos2": (R, W, 2), "row": (R,)}
            return tuple(_view(getattr(L, acc)(res), int(np.prod(shapes[row])), dt).reshape(shapes[row]) if a else None
                         for (_, acc, dt, row, _), a in zip(self._DENSE_OUTPUTS, asked))
        rows = _read_result(self, res, views)[0]
        return {key: v for (key, *_), v, a in zip(self._DENSE_OUTPUTS, rows, asked) if a or key == "attention_mask"}

    def encode_batch_dense(self, data, doc_off=None, add_special_tokens=True, want_mask=True, return_overflowing_tokens=False,
                           return_offsets_mapping=False, trim_offsets=False, return_special_tokens_mask=False, return_sequence_ids=False,
                           return_word_ids=False):
        """Batch of single sequences -> {"input_ids": uint32[n, L], "attention_mask": uint8[n, L] | None, "lengths": uint32[n]}
        with the tokenizer's truncation, template and padding applied on the device (what `encode_batch` + stacking the
        Encodings' ids / attention_mask gives in the reference).  `data` is a list of str, or packed (np.uint8[N], np.uint64[n+1]).
        return_overflowing_tokens: the overflowing parts of truncated sequences (the truncation's stride honoured) become rows
        too -- each input's kept row, then its overflowing rows, what stacking `[e] + e.overflowing` gives -- and the dict
        gains "overflow_to_sample_mapping" (uint32[R], the input of each row).  return_offsets_mapping: "offset_mapping"
        (uint32[R, L, 2], char offsets; (0, 0) for special tokens and padding).  An overflowing row longer than L is refused
        (B2TError; the reference returns it longer and unpadded); a stride not below a sequence's max_len raises ValueError.
        trim_offsets: the offset rows as the post-processor leaves them -- trimmed (ByteLevel process_offsets, every part on its
        own) where it trims offsets, unchanged where it does not; without it offsets behind a trimming post-processor raise
        UnsupportedConfig.  An added token with both lstrip and rstrip that absorbed whitespace raises UnsupportedConfig there.
        return_special_tokens_mask / return_sequence_ids / return_word_ids: "special_tokens_mask" (uint8[R, L], 1 for template
        tokens and padding), "sequence_ids" (int8[R, L], -1 = None) and "word_ids" (int32[R, L], -1 = None), as the reference's
        Encoding has them."""
        if doc_off is None:
            data, doc_off = _pack(data, np.uint64)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        doc_off = np.ascontiguousarray(doc_off, dtype=np.uint64)
        sp, keep = self.dense_spec(add_special_tokens, want_mask, return_overflowing_tokens, return_offsets_mapping, trim_offsets,
                                   return_special_tokens_mask, return_sequence_ids, return_word_ids)
        try:
            return self._dense_call("b2t_encode_batch_dense", data, doc_off, len(doc_off) - 1, sp)
        except B2TError as ex:
            if ex.code == _lib.B2T_ERR_TRUNCATION:   # the reference's stride panic, with its message
                raise ValueError(str(ex)) from None
            if ex.code == _lib.B2T_ERR_UNSUPPORTED and sp.dense_flags & _lib.DENSE_TRIM_OFFSETS:   # (the lstrip + rstrip refusal)
                raise UnsupportedConfig(str(ex)) from None
            raise

    def encode_pairs_dense(self, pairs, doc_off=None, add_special_tokens=True, want_mask=True, return_overflowing_tokens=False,
                           return_offsets_mapping=False, trim_offsets=False, return_special_tokens_mask=False, return_sequence_ids=False,
                           return_word_ids=False):
        """Batch of pairs of sequences -> {"input_ids": uint32[n, L], "token_type_ids": uint8[n, L], "attention_mask": uint8[n, L]
        | None, "lengths": uint32[n]} with the tokenizer's pair truncation, pair template and padding applied on the device
        (what `encode_batch` on pairs + stacking the Encodings' ids / type_ids / attention_mask gives in the reference).
        `pairs` is a list of (str, str), or packed (np.uint8[N], np.uint64[2n+1]): document 2p is the first sequence of
        pair p, 2p + 1 the second.  A pair that cannot be truncated raises ValueError as the reference does.
        return_overflowing_tokens / return_offsets_mapping as in encode_batch_dense: a pair gives (1 + o_x)(1 + o_y) rows for
        the parts of its two sequences, in the reference's order; without return_overflowing_tokens a stride is refused
        (UnsupportedConfig: it only shapes the overflowing parts).  trim_offsets and the row metadata as in encode_batch_dense;
        sequence ids are 0 for the pair's first sequence and 1 for its second, whatever the template order."""
        if doc_off is None:
            seqs = []
            for x in pairs:
                if not (isinstance(x, (tuple, list)) and len(x) == 2 and all(isinstance(t, str) for t in x)):
                    raise TypeError("encode_pairs_dense expects pairs (str, str)")
                seqs.extend(x)
            pairs, doc_off = _pack(seqs, np.uint64)
        data = np.ascontiguousarray(pairs, dtype=np.uint8)
        doc_off = np.ascontiguousarray(doc_off, dtype=np.uint64)
        if len(doc_off) % 2 != 1:
            raise ValueError(f"a batch of n pairs has 2n + 1 document offsets, not {len(doc_off)}")
        sp, keep = self.pair_dense_spec(add_special_tokens, want_mask, return_overflowing_tokens, return_offsets_mapping, trim_offsets,
                                        return_special_tokens_mask, return_sequence_ids, return_word_ids)
        try:
            return self._dense_call("b2t_encode_pairs_dense", data, doc_off, (len(doc_off) - 1) // 2, sp)
        except B2TError as ex:
            if ex.code == _lib.B2T_ERR_TRUNCATION:   # TruncationError::SequenceTooShort, with the reference's message
                raise ValueError(str(ex)) from None
            if ex.code == _lib.B2T_ERR_UNSUPPORTED:
                raise UnsupportedConfig(str(ex)) from None
            raise

    def _trim_tables(self):
        """per token id: leading / trailing 'G-dot' characters (the byte-level image of U+0020) of its vocabulary string"""
        if self._trim is None:
            n = max(max(self._vocab.values()), max(self._added.tokens) if self._added is not None else 0) + 1
            lead, trail = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
            for t, i in self._vocab.items():
                lead[i] = len(t) - len(t.lstrip("\u0120"))
                trail[i] = len(t) - len(t.rstrip("\u0120"))
            self._trim = (lead, trail)
        return self._trim

    def _span_spaces(self, raw, a, b):
        """leading / trailing whitespace characters of an added token's matched span (char::is_whitespace or G-dot)"""
        t = bytes(raw[a:b]).decode("utf-8", "replace")
        ws = lambda c: c == "\u0120" or self._added._class(ord(c)) == added.CLS_S
        lead = next((k for k, c in enumerate(t) if not ws(c)), len(t))
        trail = next((k for k, c in enumerate(reversed(t)) if not ws(c)), len(t))
        return lead, trail

    def _pad_all(self, out):
        """pad_encodings (utils/padding.rs:50-81); the per-sequence padding of post_process step 3 is subsumed by it"""
        pd = self._padding
        if pd is not None and out:
            target = pd["length"] if pd["length"] is not None else max(len(e) for e in out)
            m = pd["pad_to_multiple_of"]
            if m and target % m:
                target += m - target % m
            for e in out:
                e._pad(target, pd["pad_id"], pd["pad_type_id"], pd["pad_token"], pd["direction"] == "left")
        return out

    def _encode_pairs(self, inputs, offsets, word_ids, add_special_tokens):
        """Batches with pairs of sequences: the engine encodes every sequence as a row of its own; truncation, the
        post-processor and the merge of the two halves (with all combinations of their overflowing parts) follow the
        reference one input at a time (pairs.py)."""
        from . import pairs  # (pairs.py uses the post-processing rules of this module)
        seqs, first = [], []
        for x in inputs:
            first.append(len(seqs))
            if isinstance(x, str):
                seqs.append(x)
            elif isinstance(x, (tuple, list)) and len(x) == 2 and all(isinstance(t, str) for t in x):
                seqs.extend(x)
            else:
                raise UnsupportedConfig("inputs must be str or a pair (str, str)")
        first.append(len(seqs))
        data, off = _pack(seqs, np.uint64)
        be, trim = self._encode_core(data, off, _lib.WANT_OFFSETS | _lib.WANT_WORD_IDS, True)
        rp = be.row_ptr.tolist()
        ids, offs, wid = be.ids.tolist(), [tuple(o) for o in be.offsets.tolist()], be.word_ids.tolist()
        ld, tr = (trim[0].tolist(), trim[1].tolist()) if trim is not None else (None, None)

        text = be.token_text or {}

        def pe(row, type_id):
            a, b = rp[row], rp[row + 1]
            n = b - a
            p = pairs.PE(ids[a:b], [type_id] * n, wid[a:b], offs[a:b], [0] * n, [1] * n, [type_id] * n,
                         None if ld is None else ld[a:b], None if tr is None else tr[a:b])
            p.text = [text.get(i) for i in range(a, b)]
            return p

        def to_encoding(p):
            n = len(p)
            one = BatchEncoding(np.asarray(p.ids, dtype=np.uint32),
                                np.asarray(p.offsets, dtype=np.uint32).reshape(-1, 2) if offsets else None,
                                np.asarray([NO_WORD if w is None else w for w in p.words], dtype=np.uint32) if word_ids else None,
                                np.array([0, n], dtype=np.uint64), np.asarray(p.type_ids, dtype=np.uint32),
                                np.asarray(p.special, dtype=np.uint8), None,
                                np.asarray([-1 if q is None else q for q in p.seq], dtype=np.int8))
            if any(t is not None for t in p.text):
                one.token_text = {i: t for i, t in enumerate(p.text) if t is not None}
            e = Encoding(self, one, 0, n)
            if p.overflowing:
                e.overflowing = [to_encoding(o) for o in p.overflowing]
            return e

        out = []
        for i in range(len(inputs)):
            r = first[i]
            a = pe(r, 0)
            b = pe(r + 1, 1) if first[i + 1] - r == 2 else None
            out.append(to_encoding(pairs.post_process(a, b, self._template, self._truncation, add_special_tokens)))
        return self._pad_all(out)

    def _encode_list(self, docs, offsets, word_ids, add_special_tokens, is_pretokenized=False):
        if not is_pretokenized and any(not isinstance(d, str) for d in docs):
            return self._encode_pairs(docs, offsets, word_ids, add_special_tokens)
        seq_rows = None
        if is_pretokenized:
            # tokenizer/mod.rs:762-805: every word of a pre-tokenized sequence is encoded on its own (added tokens,
            # pre-tokenizer, model), its tokens keep offsets relative to the word and all get the word's index
            if any(isinstance(d, str) for d in docs):
                raise TypeError("is_pretokenized=True expects sequences of words (List[str]), not str")
            seq_rows = np.cumsum([0] + [len(d) for d in docs], dtype=np.int64)
            docs = [w for d in docs for w in d]
        try:
            data, off = _pack(docs, np.uint64)
        except AttributeError:
            raise UnsupportedConfig("only raw sequences (str), or lists of words with is_pretokenized=True, are supported; pairs are not") from None
        flags = (_lib.WANT_OFFSETS if offsets else 0) | (_lib.WANT_WORD_IDS if word_ids else 0)
        be, trim = self._encode_core(data, off, flags, True)
        if seq_rows is not None:  # rows (words) -> sequences
            wid = None
            if be.word_ids is not None:
                counts = np.diff(be.row_ptr).astype(np.int64)
                word_in_seq = np.arange(len(docs), dtype=np.int64) - np.repeat(seq_rows[:-1], np.diff(seq_rows))
                wid = np.repeat(word_in_seq, counts).astype(np.uint32)
            text = be.token_text
            be = BatchEncoding(be.ids, be.offsets, wid, be.row_ptr[seq_rows])
            be.token_text = text
        # TokenizerImpl::post_process (tokenizer/mod.rs:1265-1317): 1. truncate, 2. post-processor, 3. pad
        part_doc = np.arange(len(be.row_ptr) - 1, dtype=np.int64)
        tr = self._truncation
        if tr is not None:
            max_len = truncation_budget(tr, self._template, False, add_special_tokens)
            if tr["strategy"] == "only_second" and np.any(np.diff(be.row_ptr).astype(np.int64) > max_len):
                raise ValueError("Truncation error: Second sequence not provided")
            be, cut, part_doc = truncate_csr(be, list(trim) if trim is not None else [], max_len, tr["stride"], tr["direction"])
            trim = tuple(cut) if trim is not None else None
        be = self._finish(be, trim, add_special_tokens)
        rp = be.row_ptr.tolist()
        if tr is None:
            out = [Encoding(self, be, a, b) for a, b in zip(rp[:-1], rp[1:])]
        else:
            out, prev = [], -1
            for i, d in enumerate(part_doc.tolist()):
                enc = Encoding(self, be, rp[i], rp[i + 1])
                if d == prev:
                    out[-1].overflowing = list(out[-1].overflowing) + [enc]  # the parts of a truncated sequence follow its kept part
                else:
                    out.append(enc); prev = d
        return self._pad_all(out)

    def encode_batch(self, input, is_pretokenized=False, add_special_tokens=True):
        """tokenizer.rs:1312-1340 -> TokenizerImpl::encode_batch_char_offsets (tokenizer/mod.rs:1360-1379)."""
        return self._encode_list(list(input), True, True, add_special_tokens, is_pretokenized)

    def encode_batch_fast(self, input, is_pretokenized=False, add_special_tokens=True):
        """tokenizer.rs:1433-1461 -> encode_batch_fast (tokenizer/mod.rs:1382-1401): ids only."""
        return self._encode_list(list(input), False, False, add_special_tokens, is_pretokenized)

    def encode(self, sequence, pair=None, is_pretokenized=False, add_special_tokens=True):
        if pair is not None:
            if is_pretokenized:
                raise UnsupportedConfig("pre-tokenized pairs are not supported")
            return self._encode_list([(sequence, pair)], True, True, add_special_tokens)[0]
        return self._encode_list([sequence], True, True, add_special_tokens, is_pretokenized)[0]

    # ---- decode (tokenizer/mod.rs:935-953; host only: ids -> text is a table walk, nothing for the GPU to do)
    def decode(self, ids, skip_special_tokens=True):
        toks = []
        for i in ids:
            t = self.id_to_token(i)
            if t is None:
                continue
            if skip_special_tokens and self._added is not None and t in self._added.by_content and self._added.by_content[t].special:
                continue
            toks.append(t)
        d = self._decoder
        if d is None:
            return " ".join(toks)
        if d.get("type") == "ByteLevel":  # pre_tokenizers/byte_level.rs:156-171
            inv = _char_bytes()
            out = bytearray()
            for t in toks:
                try:
                    out.extend(inv[c] for c in t)
                except KeyError:
                    out.extend(t.encode("utf-8"))
            return out.decode("utf-8", "replace")
        if d.get("type") == "WordPiece":  # decoders/wordpiece.rs:31-61
            prefix, clean, out = d.get("prefix", "##"), d.get("cleanup", True), []
            for k, t in enumerate(toks):
                if k != 0:
                    t = t[len(prefix):] if t.startswith(prefix) else " " + t
                if clean:
                    for a, b in ((" .", "."), (" ?", "?"), (" !", "!"), (" ,", ","), (" ' ", "'"), (" n't", "n't"), (" 'm", "'m"),
                                 (" do not", " don't"), (" 's", "'s"), (" 've", "'ve"), (" 're", "'re")):
                        t = t.replace(a, b)
                out.append(t)
            return "".join(out)
        raise UnsupportedConfig(f"decoder {d.get('type')} is not supported")

    def decode_batch(self, sequences, skip_special_tokens=True):
        return [self.decode(s, skip_special_tokens) for s in sequences]

    # ---- device decode (b2t_decode_batch*): decode() of every row, on the GPU
    def _decode_ready(self):
        if self._decoder_refused is not None:
            raise UnsupportedConfig(f"device decode is not available: {self._decoder_refused}")

    @staticmethod
    def _u32_ids(ids):
        """integer ids -> uint32, ValueError for ids outside [0, 2^32) (the reference's binding takes u32)"""
        a = np.asarray(ids)
        if a.size and a.dtype.kind not in "iu":
            raise ValueError(f"ids must be integers, not {a.dtype}")
        if a.size and (int(a.min()) < 0 or int(a.max()) >= 1 << 32):
            raise ValueError("ids must lie in [0, 2^32)")
        return np.ascontiguousarray(a, dtype=np.uint32)

    def decode_batch_csr(self, ids, row_ptr, skip_special_tokens=True):
        """Rows of the token CSR (row d = ids[row_ptr[d]:row_ptr[d + 1]], as encode_batch_csr returns them) -> (text uint8,
        text_off uint64[n + 1]): row d's text is text[text_off[d]:text_off[d + 1]], exactly decode(row, skip_special_tokens)"""
        self._decode_ready()
        ids = self._u32_ids(ids).reshape(-1)
        rp = np.ascontiguousarray(row_ptr, dtype=np.uint64)
        if rp.size == 0:
            raise ValueError("row_ptr holds n_rows + 1 offsets")
        return self._decode_host(ids, rp, None, rp.size - 1, skip_special_tokens)

    def _decode_host(self, ids, row_ptr, row_len, n_rows, skip):
        L = _lib.lib()
        res = ctypes.c_void_p()
        _lib.check(L.b2t_decode_batch(self._h, ids.ctypes.data if ids.size else None, ids.size, row_ptr.ctypes.data,
                                      None if row_len is None else row_len.ctypes.data, n_rows, _lib.DECODE_SKIP_SPECIAL if skip else 0,
                                      ctypes.byref(res)))
        (text, off), _ = _read_result(self, res, lambda L, res: (_view(L.b2t_result_text(res), L.b2t_result_n_tokens(res), np.uint8),
                                                               _view(L.b2t_result_text_off(res), n_rows + 1, np.uint64)))
        return text, off

    def decode_batch_rows(self, ids, lengths=None, skip_special_tokens=True):
        """[n, L] rows of ids (numpy or torch; a CUDA tensor on the engine's device is decoded where it lies) -> n strings,
        decode(row[:lengths[i]], skip_special_tokens) each; lengths=None decodes whole rows, padding included."""
        self._decode_ready()
        torch = None
        if type(ids).__module__.startswith("torch"):
            import torch
        if torch is not None and ids.is_cuda and ids.device.index == (self._device if self._device >= 0 else torch.cuda.current_device()):
            text, off = self._decode_rows_device(torch, ids, lengths, skip_special_tokens)
        else:
            a = ids.cpu().numpy() if torch is not None else ids
            a = self._u32_ids(a)
            if a.ndim != 2:
                raise ValueError("ids must be [n, L]")
            n, w = a.shape
            if lengths is None:
                text, off = self._decode_host(a.reshape(-1), np.arange(n + 1, dtype=np.uint64) * np.uint64(w), None, n, skip_special_tokens)
            else:
                ln = self._row_lengths(lengths.cpu().numpy() if hasattr(lengths, "cpu") else lengths, n, w)
                text, off = self._decode_host(a.reshape(-1), np.arange(n, dtype=np.uint64) * np.uint64(w), ln.astype(np.uint32), n, skip_special_tokens)
        tb = text.tobytes()
        o = off.tolist()
        return [tb[o[i]:o[i + 1]].decode("utf-8") for i in range(len(o) - 1)]

    @staticmethod
    def _row_lengths(lengths, n, w):
        ln = np.asarray(lengths).reshape(-1)
        if ln.shape != (n,) or (n and (ln.dtype.kind not in "iu" or int(ln.min()) < 0 or int(ln.max()) > w)):
            raise ValueError(f"lengths must be {n} integers in [0, {w}]")
        return ln

    def _decode_rows_device(self, torch, ids, lengths, skip):
        """b2t_decode_batch_device on a CUDA tensor (int64 is narrowed on the device) -> host (text, text_off)"""
        if ids.dim() != 2:
            raise ValueError("ids must be [n, L]")
        if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
            raise ValueError(f"ids must be integers, not {ids.dtype}")
        n, w = ids.shape
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= 1 << 32):
            raise ValueError("ids must lie in [0, 2^32)")
        dev = ids.device
        ids32 = ids.to(torch.int32).contiguous()    # (the bit pattern of ids in [2^31, 2^32): unknown ids either way)
        if lengths is None:
            rp, rl = torch.arange(n + 1, device=dev, dtype=torch.int64) * w, None
        else:
            ln = torch.as_tensor(lengths, device=dev).reshape(-1)
            if ln.shape[0] != n or (n and (ln.dtype.is_floating_point or int(ln.min()) < 0 or int(ln.max()) > w)):
                raise ValueError(f"lengths must be {n} integers in [0, {w}]")
            rp, rl = torch.arange(n, device=dev, dtype=torch.int64) * w, ln.to(torch.int32).contiguous()
        L = _lib.lib()
        res = ctypes.c_void_p()
        st = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(L.b2t_decode_batch_device(self._h, ids32.data_ptr() if ids32.numel() else None, ids32.numel(), rp.data_ptr(),
                                             None if rl is None else rl.data_ptr(), n, _lib.DECODE_SKIP_SPECIAL if skip else 0, st, ctypes.byref(res)))
        try:
            nb = L.b2t_result_n_tokens(res)
            off = _device_view(torch, L.b2t_result_text_off(res), n + 1, torch.int64, dev).cpu().numpy().view(np.uint64)
            text = _device_view(torch, L.b2t_result_text(res), nb, torch.uint8, dev).cpu().numpy() if nb else np.zeros(0, np.uint8)
        finally:
            L.b2t_result_free(res)
        return text, off

    def pre_tokenize_batch(self, docs):
        """PreTokenizer seam: per document the list of (start_byte, end_byte) of its splits of the text as given (the
        normalizer and the added tokens do not apply, as with the reference's `pre_tokenizer.pre_tokenize_str`)."""
        data, off = _pack(docs, np.uint64)
        n = len(off) - 1
        L = _lib.lib()
        res = ctypes.c_void_p()
        _lib.check(L.b2t_pre_tokenize_batch(self._h, data.ctypes.data if data.size else None, off.ctypes.data, n, ctypes.byref(res)))
        (offs, rp), _ = _read_result(self, res, lambda L, res: (_view(L.b2t_result_offsets(res), 2 * L.b2t_result_n_tokens(res), np.uint32).reshape(-1, 2),
                                                          _view(L.b2t_result_row_ptr(res), n + 1, np.uint64)))
        return [[tuple(x) for x in offs[int(rp[i]):int(rp[i + 1])].tolist()] for i in range(n)]
