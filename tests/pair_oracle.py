"""TEST INFRASTRUCTURE: the plain restatement of dense pair rows (b2t_encode_pairs_dense) the tests compare the engine, the
kernels' own algebra (tests/native/dense_emul.cpp) and the shim's spec building against.  It sits beside oracle.dense_rows
(oracle/oracle.py), the single-sequence restatement, and is written the same way: straight from the reference, one pair
at a time, on Python lists."""
import numpy as np


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
