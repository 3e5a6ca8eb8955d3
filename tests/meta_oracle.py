"""TEST INFRASTRUCTURE: the plain restatement of dense rows WITH their per-position metadata (b2t_encode_batch_dense /
b2t_encode_pairs_dense with B2T_DENSE_TRIM_OFFSETS, B2T_DENSE_SPECIAL_MASK, B2T_DENSE_SEQUENCE_IDS, B2T_DENSE_WORD_IDS) that
the tests compare the engine and the kernels' own rules (tests/native/meta_emul.cpp) against.  It runs the shim's host
restatement of the reference one input at a time -- pairs.post_process (truncation with its stride, ByteLevel
process_offsets on every part of every sequence, the template, merge_with) on PEs that carry each token's leading /
trailing space counts and its word -- and flattens every input kept row first (`[e] + e.overflowing`), then pads as
overflow_oracle pads: special-tokens mask 1, sequence id and word id -1 (None) on padding."""
import numpy as np
from tokenizers_b200 import pairs


def dense_meta_rows(ids, offsets, words, row_ptr, ld=None, tr=None, *, is_pair, template, truncation, padding, add_special_tokens,
                    pad_all_rows=False):
    """TEST INFRASTRUCTURE.  ids / offsets [T, 2] / words / row_ptr: the CSR of the batch (documents 2p, 2p + 1 = pair p when
    is_pair); ld / tr: per CSR token, the leading / trailing space counts process_offsets uses (the vocabulary rule, and
    _span_spaces on an added token's matched span), or None where the template does not trim; the other arguments as
    overflow_oracle.dense_overflow_rows.
    -> (ids uint32[R, L], type ids uint8[R, L], mask uint8[R, L], lengths uint32[R], sample uint32[R], offsets uint32[R, L, 2],
    special-tokens mask uint8[R, L], sequence ids int8[R, L], word ids int32[R, L]), or the error message (as
    dense_overflow_rows)."""
    rp = [int(x) for x in row_ptr]
    per = 2 if is_pair else 1
    n_in = (len(rp) - 1) // per
    NO_WORD = 0xFFFFFFFF

    def pe(d, type_id):
        a, b = rp[d], rp[d + 1]
        n = b - a
        return pairs.PE([int(x) for x in ids[a:b]], [type_id] * n, [None if int(w) == NO_WORD else int(w) for w in words[a:b]],
                        [tuple(int(v) for v in o) for o in offsets[a:b]], [0] * n, [1] * n, [type_id] * n,
                        None if ld is None else [int(x) for x in ld[a:b]], None if tr is None else [int(x) for x in tr[a:b]])

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
