"""TEST INFRASTRUCTURE: the plain restatement of dense rows WITH overflowing parts (b2t_encode_batch_dense /
b2t_encode_pairs_dense with B2T_DENSE_OVERFLOW, B2T_DENSE_OFFSETS) that the tests compare the engine and the kernels'
own algebra (tests/native/overflow_emul.cpp) against.  It runs the shim's host restatement of the reference one input at a
time -- pairs.post_process (truncate_encodings, Encoding::truncate with its stride, the template, merge_with) on the
oracle's CSR -- and flattens every input kept row first (`[e] + e.overflowing`), then pads as pad_encodings does: to the
fixed length, or to the longest KEPT row (utils/padding.rs:50-81 looks at the top-level encodings only)."""
import numpy as np
from tokenizers_b200 import pairs


def dense_overflow_rows(ids, offsets, row_ptr, *, is_pair, template, truncation, padding, add_special_tokens, pad_all_rows=False):
    """TEST INFRASTRUCTURE.  ids / offsets [T, 2] / row_ptr: the CSR of the batch (documents 2p, 2p + 1 = pair p when
    is_pair); template: parse_post_processor's dict or None; truncation: the shim's dict (max_length, stride, strategy,
    direction) or None; padding: dict(length | None, direction, pad_id, pad_type_id, pad_to_multiple_of).
    -> (ids uint32[R, L], type ids uint8[R, L], mask uint8[R, L], lengths uint32[R], sample uint32[R], offsets uint32[R, L, 2]),
    or the error message: the reference's truncation errors (ValueError from the restatement; every distinct one the
    batch's inputs hit, joined by " | ", so that a caller can tell a batch that can only fail one way from one that holds
    both a SequenceTooShort input and a stride panic), or a row that does not fit L (the engine refuses what the reference
    returns longer).  pad_all_rows: L = the longest of ALL rows instead (no padding
    mode of the reference: the width the kernels' count pass checks)."""
    rp = [int(x) for x in row_ptr]
    per = 2 if is_pair else 1
    n_in = (len(rp) - 1) // per

    def pe(d, type_id):
        a, b = rp[d], rp[d + 1]
        n = b - a
        return pairs.PE([int(x) for x in ids[a:b]], [type_id] * n, [0] * n, [tuple(int(v) for v in o) for o in offsets[a:b]], [0] * n, [1] * n,
                        [type_id] * n)

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
        lens[r] = n
    return out, tout, mask, lens, np.asarray(sample, dtype=np.uint32), offs
