#!/usr/bin/env python
"""Throughput of dense rows with overflowing parts (B2T_DENSE_OVERFLOW [+ B2T_DENSE_OFFSETS]): sliding windows on the device.

    python tools/bench_overflow.py [--mb 64] [--steps 5] [--subset 2000]

Three workloads:
  qa_bert      extractive-QA preprocessing: a short question + a corpus context of 1-8 KB, the bert-base pipeline
               (BertNormalizer + BertPreTokenizer + WordPiece) with BertProcessing, only_second, max_length 384, stride 128,
               L = 384, offsets on;
  qa_roberta   the same with the GPT-2 style pipeline and RobertaProcessing, without offsets;
  windows      single sequences (the contexts alone), bert-base pipeline, max_length 512, stride 64, L = 512.
For each it times the pinned host path (encode_pairs_dense / encode_batch_dense) and the device entry point (per-kernel
times included) in GB/s of input and rows/s, and on a subset checks the rows against the reference wheel's encode_batch
flattened `[e] + e.overflowing` (timed at its best thread count).  Prints one JSON object."""
import argparse, ctypes, gzip, hashlib, json, os, random, subprocess, sys, tempfile, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_pairs import gpu_card, log   # noqa: E402

WORKLOADS = {  # name -> (pipeline, pairs, max_length, stride, L, offsets)
    "qa_bert": ("bert", True, 384, 128, 384, True),
    "qa_roberta": ("roberta", True, 384, 128, 384, False),
    "windows": ("bert", False, 512, 64, 512, False),
}


def tokenizer_json(pipeline):
    j = json.loads(gzip.open(os.path.join(ROOT, "assets", ("wordpiece" if pipeline == "bert" else "gpt2_style") + ".json.gz")).read().decode("utf-8"))
    v = j["model"]["vocab"]
    if pipeline == "bert":
        j["normalizer"] = {"type": "BertNormalizer", "clean_text": True, "handle_chinese_chars": True, "strip_accents": None, "lowercase": True}
        j["pre_tokenizer"] = {"type": "BertPreTokenizer"}
        j["post_processor"] = {"type": "BertProcessing", "sep": ["[SEP]", v["[SEP]"]], "cls": ["[CLS]", v["[CLS]"]]}
    else:
        j["post_processor"] = {"type": "RobertaProcessing", "sep": ["b", v["b"]], "cls": ["a", v["a"]], "trim_offsets": True, "add_prefix_space": False}
    return json.dumps(j)


def qa_inputs(mb, seed=5):
    """(question, context) pairs: contexts are 1-8 KB slices of the corpus text, questions its first words"""
    import corpus
    data, off = corpus.generate(2, seed, 0, 10_000_000, max_bytes=(mb << 20) + (1 << 20))
    text = bytes(data).decode("utf-8", "ignore")
    rng, pos, out, total = random.Random(seed), 0, [], 0
    while total < (mb << 20) and pos < len(text) - 8192:
        n = rng.randint(1024, 8192)
        ctx = text[pos:pos + n]
        pos += n
        out.append(("what about " + " ".join(ctx.split()[:4]) + "?", ctx))
        total += len(ctx.encode()) + len(out[-1][0].encode())
    return out


def flat_rows(d, pairs, offsets):
    return [d["input_ids"], d["token_type_ids"] if pairs else None, d["attention_mask"], d.get("offset_mapping") if offsets else None]


def digest(arrays):
    return hashlib.sha256(b"".join(np.ascontiguousarray(x).tobytes() for x in arrays if x is not None)).hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--subset", type=int, default=2000)
    a = ap.parse_args()
    import torch
    import corpus
    from tokenizers_b200 import Tokenizer, _lib
    corpus.build()
    L = _lib.lib()
    out = {"gpu": gpu_card(), "workloads": {}}
    inputs = qa_inputs(a.mb)
    for name, (pipeline, is_pair, max_len, stride, length, offsets) in WORKLOADS.items():
        js = tokenizer_json(pipeline)
        seqs = [s for p in inputs for s in p] if is_pair else [c for _, c in inputs]
        bs = [s.encode("utf-8") for s in seqs]
        off = np.zeros(len(bs) + 1, dtype=np.uint64); np.cumsum([len(b) for b in bs], out=off[1:])
        data = np.frombuffer(b"".join(bs), dtype=np.uint8)
        nb, n_in = int(off[-1]), len(seqs) // (2 if is_pair else 1)
        tok = Tokenizer.from_str(js, device=0)
        tok.enable_truncation(max_len, stride=stride, strategy="only_second" if is_pair else "longest_first")
        tok.enable_padding(length=length, pad_id=0)
        enc = tok.encode_pairs_dense if is_pair else tok.encode_batch_dense
        kw = dict(return_overflowing_tokens=True, return_offsets_mapping=offsets)
        h = ctypes.c_void_p()
        _lib.check(L.b2t_host_alloc(nb + 64, ctypes.byref(h)))
        pinned = np.ctypeslib.as_array(ctypes.cast(h, ctypes.POINTER(ctypes.c_uint8)), shape=(nb + 64,))
        pinned[:nb] = data
        host = enc(pinned[:nb], off, **kw)   # warm-up
        R = host["input_ids"].shape[0]
        t0 = time.perf_counter()
        for _ in range(a.steps):
            host = enc(pinned[:nb], off, **kw)
        t_host = (time.perf_counter() - t0) / a.steps
        log(name, ":", n_in, "inputs,", R, "rows,", round(nb / t_host / 1e9, 2), "GB/s host path")
        sp, keep = (tok.pair_dense_spec if is_pair else tok.dense_spec)(return_overflowing_tokens=True, return_offsets_mapping=offsets)
        d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        res = ctypes.c_void_p()
        f = L.b2t_encode_pairs_dense_device if is_pair else L.b2t_encode_batch_dense_device

        def dev_step():
            _lib.check(f(tok.handle, d_bytes.data_ptr(), nb, d_off.data_ptr(), n_in, ctypes.byref(sp), None, ctypes.byref(res)))
            assert L.b2t_result_dense_rows(res) == R
            L.b2t_result_free(res)
        dev_step()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(a.steps):
            dev_step()
        ev[1].record()
        torch.cuda.synchronize()
        t_dev = ev[0].elapsed_time(ev[1]) / 1e3 / a.steps
        L.b2t_engine_set_profiling(tok.handle, 1)
        dev_step()
        names, ms = (ctypes.c_char_p * 16)(), (ctypes.c_float * 16)()
        L.b2t_engine_last_kernels(tok.handle, names, ms, 16)
        kernels = {names[i].decode(): round(ms[i], 3) for i in range(16) if names[i]}
        L.b2t_engine_set_profiling(tok.handle, 0)
        log(name, ": device entry point", round(nb / t_dev / 1e9, 2), "GB/s", kernels)
        del d_bytes, d_off
        # the wheel on a subset: identical flattened rows, and its time at its best thread count
        k = min(a.subset, len(inputs))
        sub = inputs[:k] if is_pair else [c for _, c in inputs[:k]]
        mine = enc(sub, **kw)
        same = bool(np.array_equal(host["input_ids"][:mine["input_ids"].shape[0]], mine["input_ids"]))
        wheel = None
        try:
            import tokenizers
            best = None
            with tempfile.NamedTemporaryFile("w", suffix=".json") as fj:
                fj.write(js); fj.flush()
                for thr in ("1", "4", "16", str(os.cpu_count())):
                    r = subprocess.run([sys.executable, "-c", WHEEL_SNIPPET, fj.name, json.dumps([max_len, stride, length, is_pair, offsets])],
                                       input="\n".join(json.dumps(p) for p in sub), capture_output=True, text=True,
                                       env=dict(os.environ, RAYON_NUM_THREADS=thr), check=True)
                    t, dg = r.stdout.split()
                    best = min(best or (1e9, thr), (float(t), thr))
                    log(name, ": wheel,", thr, "threads", t, "s")
            same &= dg == digest(flat_rows(mine, is_pair, offsets))
            wheel = {"version": tokenizers.__version__, "best_threads": int(best[1]), "inputs_per_s": k / best[0], "rows_per_s": mine["input_ids"].shape[0] / best[0]}
        except ImportError:
            pass
        out["workloads"][name] = {
            "L": length, "max_length": max_len, "stride": stride, "offsets": offsets, "inputs": n_in, "rows": R, "bytes": nb,
            "host_path": {"GBps": nb / t_host / 1e9, "rows_per_s": R / t_host, "ms": t_host * 1e3},
            "device_entry_point": {"GBps": nb / t_dev / 1e9, "rows_per_s": R / t_dev, "ms": t_dev * 1e3, "kernels_ms": kernels},
            "subset": {"inputs": k, "rows": int(mine["input_ids"].shape[0]), "wheel_encode_batch": wheel, "identical": bool(same)},
        }
        L.b2t_host_free(h)
        del tok
    print(json.dumps(out))


# the wheel in a process of its own (its thread count is fixed when its pool starts): inputs as JSON lines on stdin ->
# "seconds sha256(flattened ids [, type ids], mask [, offsets])"
WHEEL_SNIPPET = r"""
import sys, json, time, hashlib, numpy as np, tokenizers
tok = tokenizers.Tokenizer.from_file(sys.argv[1]); max_len, stride, L, is_pair, offsets = json.loads(sys.argv[2])
tok.enable_truncation(max_len, stride=stride, strategy="only_second" if is_pair else "longest_first"); tok.enable_padding(length=L, pad_id=0)
inputs = [json.loads(l) for l in sys.stdin.read().splitlines()]
inputs = [tuple(x) for x in inputs] if is_pair else inputs
tok.encode_batch(inputs[:50])
t0 = time.perf_counter(); encs = tok.encode_batch(inputs); t = time.perf_counter() - t0
rows = [x for e in encs for x in [e] + list(e.overflowing)]
R = len(rows)
arrs = [np.array([x.ids for x in rows], dtype=np.uint32).reshape(R, L)]
if is_pair: arrs.append(np.array([x.type_ids for x in rows], dtype=np.uint8).reshape(R, L))
arrs.append(np.array([x.attention_mask for x in rows], dtype=np.uint8).reshape(R, L))
if offsets: arrs.append(np.array([x.offsets for x in rows], dtype=np.uint32).reshape(R, L, 2))
print(t, hashlib.sha256(b"".join(np.ascontiguousarray(x).tobytes() for x in arrs)).hexdigest())
"""

if __name__ == "__main__":
    main()
