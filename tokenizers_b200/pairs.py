"""Post-processing for batches that contain PAIRS of sequences (EncodeInput::Dual): the per-input path.

The vectorised CSR path of tokenizer.py covers single sequences; a pair needs the reference's combinatorial handling of
overflowing parts (every part of the first sequence with every part of the second), which is restated here on plain
Python lists, one input at a time:
    TokenizerImpl::post_process            tokenizer/mod.rs:1265-1317   truncate -> post-processor -> (pad: in tokenizer.py)
    truncate_encodings                      utils/truncation.rs:70-160    longest_first / only_first / only_second
    Encoding::truncate / merge_with         tokenizer/encoding.rs:307-388, 408-463
    PostProcessor::process                  tokenizer/mod.rs:126-148     sequence ids, type ids, merge of the pieces
    templates as piece lists                processors/template.rs:544-643, bert.rs:51-, roberta.rs:66-
The rules both paths share (truncation spans, the special-token count, offset trimming) live in tokenizer.py.
All tokenization still happens in the engine: this module only rearranges its output.
"""
import copy
import numpy as np
from .tokenizer import trim_spans, truncation_budget, truncation_spans


class PE:
    """A plain-Python Encoding.  words: None for special tokens; seq: index of the sequence a token belongs to or None;
    ld / tr: leading / trailing space counts of the token's text (for offset trimming), or None."""
    __slots__ = ("ids", "type_ids", "words", "offsets", "special", "attn", "seq", "text", "ld", "tr", "overflowing")

    def __init__(self, ids=(), type_ids=(), words=(), offsets=(), special=(), attn=(), seq=(), ld=None, tr=None):
        self.ids, self.type_ids, self.words, self.offsets = list(ids), list(type_ids), list(words), list(offsets)
        self.special, self.attn, self.seq = list(special), list(attn), list(seq)
        self.text = [None] * len(self.ids)  # token text where it is not the vocabulary string (lstrip / rstrip added tokens)
        self.ld, self.tr = (None if ld is None else list(ld)), (None if tr is None else list(tr))
        self.overflowing = []

    def __len__(self):
        return len(self.ids)

    def slice(self, a, b):
        p = PE(self.ids[a:b], self.type_ids[a:b], self.words[a:b], self.offsets[a:b], self.special[a:b], self.attn[a:b], self.seq[a:b],
               None if self.ld is None else self.ld[a:b], None if self.tr is None else self.tr[a:b])
        p.text = self.text[a:b]
        return p

    def clone(self):
        return copy.deepcopy(self)


def special_piece(token_id, type_id):
    return PE([token_id], [type_id], [None], [(0, 0)], [1], [1], [None])


def truncate(pe, max_len, stride, direction):
    """Encoding::truncate (encoding.rs:307-388), in place"""
    if max_len >= len(pe):
        return
    spans = truncation_spans(len(pe), max_len, stride, direction)
    new = pe.slice(*spans[0])
    new.overflowing = [pe.slice(a, b) for a, b in spans[1:]]
    for f in PE.__slots__:
        setattr(pe, f, getattr(new, f))


def truncate_pair(a, b, tr):
    """truncate_encodings (utils/truncation.rs:70-160); b may be None"""
    max_len, stride, direction, strategy = tr["max_length"], tr["stride"], tr["direction"], tr["strategy"]
    if max_len == 0:
        truncate(a, 0, stride, direction)
        if b is not None:
            truncate(b, 0, stride, direction)
        return
    total = len(a) + (len(b) if b is not None else 0)
    if total <= max_len:
        return
    to_remove = total - max_len
    if strategy == "longest_first":
        if b is None:
            truncate(a, total - to_remove, stride, direction)
            return
        n1, n2, swap = len(a), len(b), False
        if n1 > n2:
            n1, n2, swap = n2, n1, True
        n2 = n1 if n1 > max_len else max(n1, max_len - n1)
        if n1 + n2 > max_len:
            n1 = max_len // 2
            n2 = n1 + max_len % 2
        if swap:
            n1, n2 = n2, n1
        truncate(a, n1, stride, direction)
        truncate(b, n2, stride, direction)
        return
    target = a if strategy == "only_first" else b
    if target is None:
        raise ValueError("Truncation error: Second sequence not provided")
    if len(target) > to_remove:
        truncate(target, len(target) - to_remove, stride, direction)
    else:
        raise ValueError("Truncation error: Sequence to truncate too short to respect the provided max_length")


def merge_with(acc, pair):
    """Encoding::merge_with(pair, growing_offsets = false) (encoding.rs:408-463), in place on acc"""
    over = []
    for so in acc.overflowing:
        n = so.clone(); merge_with(n, pair.clone()); over.append(n)
        for oo in pair.overflowing:
            n = so.clone(); merge_with(n, oo.clone()); over.append(n)
    for oo in pair.overflowing:
        n = acc.clone(); merge_with(n, oo.clone()); over.append(n)
    for f in ("ids", "type_ids", "words", "offsets", "special", "attn", "seq", "text"):
        getattr(acc, f).extend(getattr(pair, f))
    if acc.ld is not None and pair.ld is not None:
        acc.ld.extend(pair.ld); acc.tr.extend(pair.tr)
    else:
        acc.ld = acc.tr = None
    acc.overflowing = over


def trim(pe, add_prefix_space):
    """trim_spans on one encoding and its overflowing parts; the encoding's first token is the first of its sequence"""
    for o in pe.overflowing:
        trim(o, add_prefix_space)
    if pe.ld is None or not pe.ids:
        return
    first = np.arange(len(pe)) == 0
    pe.offsets = [tuple(o) for o in trim_spans(pe.offsets, pe.ld, pe.tr, first, add_prefix_space).tolist()]


def post_process(a, b, template, truncation, add_special_tokens):
    """TokenizerImpl::post_process steps 1 and 2 for one input (b is None for a single sequence) -> merged PE"""
    is_pair = b is not None
    pieces = None
    if template is not None:
        pieces = template["pair"] if is_pair else template["single"]
        if is_pair and pieces is None:
            raise ValueError("the post-processor has no template for pairs of sequences")
    if truncation is not None:
        truncate_pair(a, b, dict(truncation, max_length=truncation_budget(truncation, template, is_pair, add_special_tokens)))
    seqs = [a] + ([b] if is_pair else [])
    for i, e in enumerate(seqs):  # PostProcessor::process (mod.rs:137-144) / default_process: sequence ids, type ids
        for x in [e] + e.overflowing:
            x.seq = [i] * len(x)
        e.type_ids = [i] * len(e)
    if template is not None and template["trim"] is not None:
        for e in seqs:
            trim(e, template["trim"])
    if pieces is None:
        pieces = [("seq", 0, 0), ("seq", 1, 1)] if is_pair else [("seq", 0, 0)]
    acc = PE(ld=[], tr=[])
    for kind, v, t in pieces:
        if kind == "seq":
            e = seqs[v]
            e.type_ids = [t] * len(e)  # the kept part takes the piece's type id; overflowing parts keep their own ...
            if add_special_tokens and template is not None and template.get("overflow_type") is not None:  # ... unless the wrapping rewrites them
                for o in e.overflowing:
                    o.type_ids = [template["overflow_type"]] * len(o)
            merge_with(acc, e)
        elif add_special_tokens:
            merge_with(acc, special_piece(v, t))
    return acc
