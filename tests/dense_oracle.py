"""TEST INFRASTRUCTURE: the plain restatements of dense rows the tests compare the engine, the kernels run on the host
(tests/native/dense_emul.cpp) and the shim's spec building against.  They sit beside oracle.dense_rows (oracle/oracle.py),
the single-sequence restatement:
  pair_keep, dense_pair_rows   pairs without overflowing parts, written straight from the reference one pair at a time on
                               Python lists -- a second implementation of the pair truncation, independent of the shim's;
  dense_meta_rows              every row the reference's post-processing makes, through the shim's host restatement
                               (pairs.post_process), with overflowing parts, offsets and the per-position metadata."""
import numpy as np
from tokenizers_b200 import pairs


def pair_keep(n1, n2, budget, strategy):
    """TEST INFRASTRUCTURE.  Plain restatement of truncate_encodings on a pair (utils/truncation.rs:70-162), kept parts only:
    n1, n2 tokens, `budget` tokens for both (None = no truncation), strategy "longest_first" | "only_first" | "only_second"
    -> (kept n1, kept n2), or None where the reference fails with TruncationError::SequenceTooShort."""
    if budget is None:
        return n1, n2
    if budget == 0:   # truncation.rs:75-81: both sequences are cut to nothing, whatever the strategy
        return 0, 0
    if n1 + n2 <= budget:
        return n1, n2
    if strategy == "longest_first":
        short, long_ = sorted((n1, n2))
        keep_long = short if short > budget else max(short, budget - short)
        keep_short = short
        if keep_short + keep_long > budget:
            keep_short = budget // 2
            keep_long = keep_short + budget % 2
        k1, k2 = (keep_long, keep_short) if n1 > n2 else (keep_short, keep_long)
        return min(n1, k1), min(n2, k2)   # Encoding::truncate (tokenizer/encoding.rs:307-388) never lengthens
    to_remove = n1 + n2 - budget
    target = n1 if strategy == "only_first" else n2
    if target <= to_remove:
        return None
    return (n1 - to_remove, n2) if strategy == "only_first" else (n1, n2 - to_remove)


def dense_pair_rows(ids, row_ptr, *, length, pad_to_multiple_of, max_length, strategy, truncate_left, pad_id, pad_type_id, pad_left, pieces):
    """TEST INFRASTRUCTURE.  Plain restatement of what the reference does to a batch of PAIRS after the model (document 2p of
    the CSR is the first sequence of pair p, 2p + 1 the second):
      truncation of the pair to max_length - the special tokens of `pieces` (tokenizer/mod.rs:1272-1283; pair_keep above;
      direction left keeps the last tokens, tokenizer/encoding.rs:307-388);
      the template `pieces` = [("special", id, type id) | ("seq", 0 for A / 1 for B, type id)] in order (processors/
      template.rs:544-643 apply_template: every token of a sequence takes its piece's type id);
      pad_encodings (utils/padding.rs:50-81): pad id, pad type id, attention mask 0.
    max_length 0 = no truncation.  -> (ids uint32[n, L], type ids uint8[n, L], attention_mask uint8[n, L], lengths uint32[n]);
    raises ValueError for a pair that cannot be truncated, or a row that does not fit a fixed length."""
    n = (len(row_ptr) - 1) // 2
    n_special = sum(1 for p in pieces if p[0] == "special")
    budget = max_length - n_special if max_length else None
    rows = []
    for p in range(n):
        seqs = [list(ids[int(row_ptr[2 * p + i]):int(row_ptr[2 * p + i + 1])]) for i in (0, 1)]
        keep = pair_keep(len(seqs[0]), len(seqs[1]), budget, strategy)
        if keep is None:
            raise ValueError("Truncation error: Sequence to truncate too short to respect the provided max_length")
        for i in (0, 1):
            s = seqs[i]
            seqs[i] = s[len(s) - keep[i]:] if truncate_left else s[:keep[i]]
        row, types = [], []
        for kind, v, t in pieces:
            part = [v] if kind == "special" else seqs[v]
            row += part
            types += [t] * len(part)
        rows.append((row, types))
    L = length if length else max((len(r) for r, _ in rows), default=0)
    if pad_to_multiple_of and L % pad_to_multiple_of:
        L += pad_to_multiple_of - L % pad_to_multiple_of
    out = np.full((n, L), pad_id, dtype=np.uint32)
    tout = np.full((n, L), pad_type_id, dtype=np.uint8)
    mask = np.zeros((n, L), dtype=np.uint8)
    lens = np.zeros(n, dtype=np.uint32)
    for p, (r, t) in enumerate(rows):
        if len(r) > L:
            raise ValueError(f"pair {p} has {len(r)} tokens, dense length is {L}")
        a = L - len(r) if pad_left else 0
        out[p, a:a + len(r)] = r
        tout[p, a:a + len(r)] = t
        mask[p, a:a + len(r)] = 1
        lens[p] = len(r)
    return out, tout, mask, lens


def dense_meta_rows(ids, offsets, words, row_ptr, ld=None, tr=None, *, is_pair, template, truncation, padding, add_special_tokens,
                    pad_all_rows=False):
    """TEST INFRASTRUCTURE.  Plain restatement of dense rows with overflowing parts, offsets and their per-position metadata
    (b2t_encode_batch_dense / b2t_encode_pairs_dense with B2T_DENSE_OVERFLOW, B2T_DENSE_OFFSETS, B2T_DENSE_TRIM_OFFSETS,
    B2T_DENSE_SPECIAL_MASK, B2T_DENSE_SEQUENCE_IDS, B2T_DENSE_WORD_IDS).  It runs the shim's host restatement of the
    reference one input at a time -- pairs.post_process (truncate_encodings, Encoding::truncate with its stride, ByteLevel
    process_offsets on every part of every sequence, the template, merge_with) -- and flattens every input kept row first
    (`[e] + e.overflowing`), then pads as pad_encodings does: to the fixed length, or to the longest KEPT row
    (utils/padding.rs:50-81 looks at the top-level encodings only); special-tokens mask 1, sequence id and word id -1
    (None) on padding.
    ids / offsets [T, 2] / words / row_ptr: the CSR of the batch (documents 2p, 2p + 1 = pair p when is_pair; words None: no
    word ids); ld / tr: per CSR token, the leading / trailing space counts process_offsets uses (the vocabulary rule, and
    _span_spaces on an added token's matched span), or None where the template does not trim; template:
    parse_post_processor's dict or None; truncation: the shim's dict (max_length, stride, strategy, direction) or None;
    padding: dict(length | None, direction, pad_id, pad_type_id, pad_to_multiple_of).  pad_all_rows: L = the longest of ALL
    rows instead (no padding mode of the reference: the width the kernels' count pass checks).
    -> (ids uint32[R, L], type ids uint8[R, L], mask uint8[R, L], lengths uint32[R], sample uint32[R], offsets uint32[R, L, 2],
    special-tokens mask uint8[R, L], sequence ids int8[R, L], word ids int32[R, L]), or the error message: the reference's
    truncation errors (ValueError from the restatement; every distinct one the batch's inputs hit, joined by " | ", so that
    a caller can tell a batch that can only fail one way from one that holds both a SequenceTooShort input and a stride
    panic), or a row that does not fit L (the engine refuses what the reference returns longer)."""
    rp = [int(x) for x in row_ptr]
    per = 2 if is_pair else 1
    n_in = (len(rp) - 1) // per
    NO_WORD = 0xFFFFFFFF

    def pe(d, type_id):
        a, b = rp[d], rp[d + 1]
        n = b - a
        wd = [0] * n if words is None else [None if int(w) == NO_WORD else int(w) for w in words[a:b]]
        return pairs.PE([int(x) for x in ids[a:b]], [type_id] * n, wd, [tuple(int(v) for v in o) for o in offsets[a:b]], [0] * n, [1] * n,
                        [type_id] * n, None if ld is None else [int(x) for x in ld[a:b]], None if tr is None else [int(x) for x in tr[a:b]])

    rows, sample, errors = [], [], []
    for p in range(n_in):
        a = pe(per * p, 0)
        b = pe(2 * p + 1, 1) if is_pair else None
        try:
            m = pairs.post_process(a, b, template, truncation, add_special_tokens)
        except ValueError as ex:
            if str(ex) not in errors:
                errors.append(str(ex))
            continue
        for e in [m] + m.overflowing:
            rows.append(e); sample.append(p)
    if errors:
        return " | ".join(errors)
    kept = [len(rows[k]) for k in range(len(rows)) if k == 0 or sample[k] != sample[k - 1]]
    L = padding["length"] if padding["length"] is not None else max(kept, default=0)
    if pad_all_rows:
        L = max((len(e) for e in rows), default=0)
    mult = padding.get("pad_to_multiple_of") or 0
    if mult and L % mult:
        L += mult - L % mult
    R = len(rows)
    out = np.full((R, L), padding["pad_id"], dtype=np.uint32)
    tout = np.full((R, L), padding["pad_type_id"], dtype=np.uint8)
    mask = np.zeros((R, L), dtype=np.uint8)
    offs = np.zeros((R, L, 2), dtype=np.uint32)
    lens = np.zeros(R, dtype=np.uint32)
    special = np.ones((R, L), dtype=np.uint8)
    seq = np.full((R, L), -1, dtype=np.int8)
    wid = np.full((R, L), -1, dtype=np.int32)
    for r, e in enumerate(rows):
        n = len(e)
        if n > L:
            return f"row {r} of {n} tokens does not fit the dense length {L}"
        s = L - n if padding["direction"] == "left" else 0
        out[r, s:s + n] = e.ids
        tout[r, s:s + n] = e.type_ids
        mask[r, s:s + n] = 1
        if n:
            offs[r, s:s + n] = np.asarray(e.offsets, dtype=np.uint32).reshape(n, 2)
        special[r, s:s + n] = e.special
        seq[r, s:s + n] = [-1 if q is None else q for q in e.seq]
        wid[r, s:s + n] = [-1 if w is None else w for w in e.words]
        lens[r] = n
    return out, tout, mask, lens, np.asarray(sample, dtype=np.uint32), offs, special, seq, wid
