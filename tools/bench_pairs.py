#!/usr/bin/env python
"""Throughput of dense pair rows (b2t_encode_pairs_dense*): consecutive documents of the synthetic corpus paired up,
pair truncation + pair template + padding on the device, [n_pairs, L] ids / type ids / mask back.

    python tools/bench_pairs.py [--mb 256] [--steps 5] [--subset 20000]

Two workloads: the bert-base pipeline (BertNormalizer + BertPreTokenizer + WordPiece) with BertProcessing at L = 128, and
the GPT-2 style pipeline with RobertaProcessing at L = 256, both longest_first.  For each it times the pinned host path
(Tokenizer.encode_pairs_dense) and the device entry point (b2t_encode_pairs_dense_device, per-kernel times included), and
on a subset of pairs the per-input path (Tokenizer.encode_batch on the pairs, pairs.py) and the reference wheel's
encode_batch at its best thread count, checking that all of them give identical stacked rows.  Prints one JSON object."""
import argparse, ctypes, gzip, json, os, subprocess, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))


def gpu_card():
    """name and power limit of GPU 0 (part of every number this prints)"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"name": out[0], "power_limit_w": float(out[1])}
    except Exception:
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None}


def workload(name):
    j = json.loads(gzip.open(os.path.join(ROOT, "assets", ("wordpiece" if name == "bert" else "gpt2_style") + ".json.gz")).read().decode("utf-8"))
    v = j["model"]["vocab"]
    if name == "bert":
        j["normalizer"] = {"type": "BertNormalizer", "clean_text": True, "handle_chinese_chars": True, "strip_accents": None, "lowercase": True}
        j["pre_tokenizer"] = {"type": "BertPreTokenizer"}
        j["post_processor"] = {"type": "BertProcessing", "sep": ["[SEP]", v["[SEP]"]], "cls": ["[CLS]", v["[CLS]"]]}
        return json.dumps(j), 4, 128
    j["post_processor"] = {"type": "RobertaProcessing", "sep": ["b", v["b"]], "cls": ["a", v["a"]], "trim_offsets": True, "add_prefix_space": False}
    return json.dumps(j), 2, 256


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def stack(encs, n):
    return (np.array([e.ids for e in encs], dtype=np.uint32).reshape(n, -1), np.array([e.type_ids for e in encs], dtype=np.uint8).reshape(n, -1),
            np.array([e.attention_mask for e in encs], dtype=np.uint8).reshape(n, -1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--subset", type=int, default=20000)
    a = ap.parse_args()
    import torch
    import corpus
    from tokenizers_b200 import Tokenizer, _lib
    corpus.build()
    L = _lib.lib()
    out = {"gpu": gpu_card(), "workloads": {}}
    for name in ("bert", "roberta"):
        js, kind, length = workload(name)
        data, off = corpus.generate(kind, 5, 0, 10_000_000, max_bytes=a.mb << 20)
        if (len(off) - 1) % 2:
            off = off[:-1]
            data = data[:int(off[-1])]
        n_pairs, nb = (len(off) - 1) // 2, int(off[-1])
        log(name, ":", n_pairs, "pairs,", nb, "bytes")
        tok = Tokenizer.from_str(js, device=0)
        tok.enable_truncation(length, strategy="longest_first")
        tok.enable_padding(length=length, pad_id=0)
        # pinned host path
        h = ctypes.c_void_p()
        _lib.check(L.b2t_host_alloc(nb + 64, ctypes.byref(h)))
        pinned = np.ctypeslib.as_array(ctypes.cast(h, ctypes.POINTER(ctypes.c_uint8)), shape=(nb + 64,))
        pinned[:nb] = data
        tok.encode_pairs_dense(pinned[:nb], off, want_mask=True)   # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.steps):
            host = tok.encode_pairs_dense(pinned[:nb], off, want_mask=True)
        t_host = (time.perf_counter() - t0) / a.steps
        log(name, ": encode_pairs_dense", round(nb / t_host / 1e9, 2), "GB/s")
        # device entry point, per-kernel times
        sp, keep = tok.pair_dense_spec()
        d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        res = ctypes.c_void_p()

        def dev_step():
            _lib.check(L.b2t_encode_pairs_dense_device(tok.handle, d_bytes.data_ptr(), nb, d_off.data_ptr(), n_pairs, ctypes.byref(sp), None, ctypes.byref(res)))
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
        # the per-input path and the wheel on a subset, all three stacked rows identical
        k = min(a.subset, n_pairs)
        sub_off = off[:2 * k + 1]
        docs = corpus.to_strings(data[:int(sub_off[-1])], sub_off)
        pairs = list(zip(docs[0::2], docs[1::2]))
        dense = tok.encode_pairs_dense(pairs)
        t0 = time.perf_counter()
        st = stack(tok.encode_batch(pairs), k)
        t_pairs_py = time.perf_counter() - t0
        log(name, ": encode_batch on", k, "pairs", round(t_pairs_py, 1), "s")
        same = all(np.array_equal(x, y) for x, y in zip(st, (dense["input_ids"], dense["token_type_ids"], dense["attention_mask"])))
        same &= np.array_equal(host["input_ids"][:k], dense["input_ids"]) and np.array_equal(host["token_type_ids"][:k], dense["token_type_ids"])
        wheel = None
        try:
            import tokenizers
            import tempfile
            best = None
            with tempfile.NamedTemporaryFile("w", suffix=".json") as f:   # (the tokenizer.json is too long for an argument)
                f.write(js); f.flush()
                for thr in ("1", "4", "16", str(os.cpu_count())):
                    r = subprocess.run([sys.executable, "-c", WHEEL_SNIPPET, f.name, str(length)], input="\n".join(json.dumps(p) for p in pairs),
                                       capture_output=True, text=True, env=dict(os.environ, RAYON_NUM_THREADS=thr), check=True)
                    t, digest = r.stdout.split()
                    best = min(best or (1e9, thr), (float(t), thr))
                    log(name, ": wheel,", thr, "threads", t, "s")
            import hashlib
            same &= digest == hashlib.sha256(b"".join(np.ascontiguousarray(x).tobytes() for x in st)).hexdigest()
            wheel = {"version": tokenizers.__version__, "best_threads": int(best[1]), "pairs_per_s": k / best[0]}
        except ImportError:
            pass
        sub_b = int(sub_off[-1])
        out["workloads"][name] = {
            "L": length, "pairs": n_pairs, "bytes": nb,
            "encode_pairs_dense": {"GBps": nb / t_host / 1e9, "pairs_per_s": n_pairs / t_host, "ms": t_host * 1e3},
            "encode_pairs_dense_device": {"GBps": nb / t_dev / 1e9, "pairs_per_s": n_pairs / t_dev, "ms": t_dev * 1e3, "kernels_ms": kernels},
            "subset": {"pairs": k, "bytes": sub_b, "encode_batch_pairs_per_s": k / t_pairs_py, "wheel_encode_batch": wheel, "identical": bool(same)},
        }
        L.b2t_host_free(h)
        del tok
    print(json.dumps(out))


# the wheel in a process of its own (its thread count is fixed when its pool starts): pairs as JSON lines on stdin ->
# "seconds sha256(stacked ids, type ids, mask)"
WHEEL_SNIPPET = r"""
import sys, json, time, hashlib, numpy as np, tokenizers
tok = tokenizers.Tokenizer.from_file(sys.argv[1]); L = int(sys.argv[2])
tok.enable_truncation(L, strategy="longest_first"); tok.enable_padding(length=L, pad_id=0)
pairs = [tuple(json.loads(l)) for l in sys.stdin.read().splitlines()]
tok.encode_batch(pairs[:100])
t0 = time.perf_counter(); encs = tok.encode_batch(pairs); t = time.perf_counter() - t0
n = len(pairs)
st = (np.array([e.ids for e in encs], dtype=np.uint32).reshape(n, -1), np.array([e.type_ids for e in encs], dtype=np.uint8).reshape(n, -1),
      np.array([e.attention_mask for e in encs], dtype=np.uint8).reshape(n, -1))
print(t, hashlib.sha256(b"".join(np.ascontiguousarray(x).tobytes() for x in st)).hexdigest())
"""

if __name__ == "__main__":
    main()
