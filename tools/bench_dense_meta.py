#!/usr/bin/env python
"""Cost of the dense row metadata (B2T_DENSE_TRIM_OFFSETS, _SPECIAL_MASK, _SEQUENCE_IDS, _WORD_IDS) on the QA workload.

    python tools/bench_dense_meta.py [--mb 64] [--steps 5]

bench_overflow's qa_roberta (a question + a 1-8 KB corpus context, the GPT-2 style pipeline with RobertaProcessing,
only_second, max_length 384, stride 128, L = 384, overflowing parts) through the device entry point, three ways:
  offsets      offset rows without trimming (B2T_DENSE_OFFSETS through the raw ABI: the shim refuses untrimmed offsets
               behind RobertaProcessing);
  trimmed      B2T_DENSE_OFFSETS | B2T_DENSE_TRIM_OFFSETS;
  all          trimmed offsets + special-tokens mask + sequence ids + word ids.
For each: the call in GB/s of input (CUDA events around whole calls) and the row kernel's time (the engine's per-kernel
events).  The three results must agree on ids, type ids, mask and sample map.  Prints one JSON object, with the card name
and power limit read in the same run."""
import argparse, ctypes, json, os, sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_pairs import gpu_card, log                    # noqa: E402
from bench_overflow import qa_inputs, tokenizer_json     # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import corpus
    from tokenizers_b200 import Tokenizer, _lib
    corpus.build()
    L = _lib.lib()
    inputs = qa_inputs(a.mb)
    seqs = [s for p in inputs for s in p]
    bs = [s.encode("utf-8") for s in seqs]
    off = np.zeros(len(bs) + 1, dtype=np.uint64); np.cumsum([len(b) for b in bs], out=off[1:])
    data = np.frombuffer(b"".join(bs), dtype=np.uint8)
    nb, n_in = int(off[-1]), len(inputs)
    tok = Tokenizer.from_str(tokenizer_json("roberta"), device=0)
    tok.enable_truncation(384, stride=128, strategy="only_second")
    tok.enable_padding(length=384, pad_id=0)
    d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    variants = {
        "offsets": (dict(return_overflowing_tokens=True), _lib.DENSE_OFFSETS),
        "trimmed": (dict(return_overflowing_tokens=True, return_offsets_mapping=True, trim_offsets=True), 0),
        "all": (dict(return_overflowing_tokens=True, return_offsets_mapping=True, trim_offsets=True, return_special_tokens_mask=True,
                     return_sequence_ids=True, return_word_ids=True), 0),
    }
    out = {"gpu": gpu_card(), "workload": "qa_roberta", "inputs": n_in, "bytes": nb, "L": 384, "max_length": 384, "stride": 128, "variants": {}}
    res = ctypes.c_void_p()
    digests = set()
    for name, (kw, extra) in variants.items():
        sp, keep = tok.pair_dense_spec(**kw)
        sp.dense_flags |= extra

        def step():
            _lib.check(L.b2t_encode_pairs_dense_device(tok.handle, d_bytes.data_ptr(), nb, d_off.data_ptr(), n_in, ctypes.byref(sp), None, ctypes.byref(res)))
        step()
        R, W = L.b2t_result_dense_rows(res), L.b2t_result_dense_length(res)
        torch.cuda.synchronize()
        cells = R * W

        def dev(ptr, count, dtype):
            h = np.empty(count, dtype=dtype)
            ctypes.CDLL("libcudart.so").cudaMemcpy(ctypes.c_void_p(h.ctypes.data), ctypes.c_void_p(ptr), ctypes.c_size_t(h.nbytes), 2)
            return h
        digests.add(hash((dev(L.b2t_result_dense_ids(res), cells, np.uint32).tobytes(), dev(L.b2t_result_type_ids(res), cells, np.uint8).tobytes(),
                          dev(L.b2t_result_attention_mask(res), cells, np.uint8).tobytes(), dev(L.b2t_result_row_sample(res), R, np.uint32).tobytes())))
        L.b2t_result_free(res)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(a.steps):
            step(); L.b2t_result_free(res)
        ev[1].record()
        torch.cuda.synchronize()
        t = ev[0].elapsed_time(ev[1]) / 1e3 / a.steps
        rows_ms = []
        L.b2t_engine_set_profiling(tok.handle, 1)
        for _ in range(a.steps):
            step()
            names, ms = (ctypes.c_char_p * 16)(), (ctypes.c_float * 16)()
            L.b2t_engine_last_kernels(tok.handle, names, ms, 16)
            L.b2t_result_free(res)
            rows_ms.append(sum(ms[i] for i in range(16) if names[i] and names[i].decode().startswith("dense_pair_rows")))
        L.b2t_engine_set_profiling(tok.handle, 0)
        out["variants"][name] = {"dense_flags": int(sp.dense_flags), "rows": R, "cells": cells, "call_ms": t * 1e3, "GBps": nb / t / 1e9,
                                 "row_kernel_ms_median": float(np.median(rows_ms)), "row_kernel_ms_min": float(min(rows_ms))}
        log(name, ":", R, "rows,", round(nb / t / 1e9, 2), "GB/s, row kernel", round(float(np.median(rows_ms)), 3), "ms")
    out["same_rows"] = len(digests) == 1
    print(json.dumps(out))


if __name__ == "__main__":
    main()
