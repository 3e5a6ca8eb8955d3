#!/usr/bin/env python
"""Device decode (b2t_decode_batch_device, b2t_decode_batch) throughput.

    python tools/bench_decode.py [--mb 1024] [--steps 5] [--wheel-docs 20000]

Workloads, every path checked for equal outputs:
  (a) gpt2_roundtrip  the bench corpus (GPT-2 style, --mb MiB) encoded on the device, its token CSR decoded device-resident
                      with the ByteLevel decoder; the text must equal the corpus bytes and text_off its document offsets
  (b) gen_rows        [B, 2048] rows cut from those ids with random lengths (some rows end inside a character), decoded
                      with row lengths
  (c) wordpiece       the WordPiece corpus with the WordPiece decoder (cleanup=True), its CSR decoded
For each: the device entry point (CUDA events around whole calls), the host entry point (wall clock, host ids in, host
text out), the engine's per-kernel times (its records of the host's reads between kernels, *_read, are reported apart and left out of the
kernel time), the tokens decoded (with row lengths: their sum, not the ids of the padded rows), the roofline share of the bytes the algorithm moves (ids and row offsets read,
text and text offsets written) over the kernels' time against 3.35 TB/s, and the reference wheel's decode_batch on the
first --wheel-docs rows (its default rayon pool: every core).  Prints one JSON object with the card name and power limit."""
import argparse, ctypes, json, os, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_pairs import gpu_card, log     # noqa: E402
from bench import gen_corpus, KIND, SEED  # noqa: E402

HBM_TBS = 3.35


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--wheel-docs", type=int, default=20000)
    a = ap.parse_args()
    import torch
    from tokenizers_b200 import Tokenizer, _lib
    from tokenizers_b200.tokenizer import _device_view
    L = _lib.lib()
    try:
        import tokenizers as wheel
    except Exception:
        wheel = None
    out = {"gpu": gpu_card(), "hbm_tb_s": HBM_TBS, "workloads": {}}
    stream = torch.cuda.current_stream().cuda_stream

    def tokenizer(asset, decoder):
        import gzip
        j = json.loads(gzip.open(os.path.join(ROOT, "assets", asset + ".json.gz")).read().decode("utf-8"))
        j["decoder"] = decoder
        return json.dumps(j)

    def encode(tok, cfg):
        buf = np.empty((a.mb << 20) + (1 << 20), dtype=np.uint8)
        n, off = gen_corpus(KIND[cfg], SEED[cfg], 0, (a.mb << 20) // 300, a.mb << 20, buf)
        data = buf[:n]
        d_bytes = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        res = ctypes.c_void_p()
        _lib.check(L.b2t_encode_batch_device(tok.handle, d_bytes.data_ptr(), n, d_off.data_ptr(), len(off) - 1, 0, None, ctypes.byref(res)))
        T = L.b2t_result_n_tokens(res)
        dev = d_bytes.device
        ids = _device_view(torch, L.b2t_result_ids(res), T, torch.int32, dev).clone()   # (u32 ids as int32 words)
        rp = _device_view(torch, L.b2t_result_row_ptr(res), len(off), torch.int64, dev).clone()
        L.b2t_result_free(res)
        return data, off, d_bytes[:n], ids, rp

    def run(name, tok, ids, rp, rl, n_rows, check):
        """device and host entry points on the same rows; check(text, text_off) on the device result"""
        res = ctypes.c_void_p()

        def call():
            _lib.check(L.b2t_decode_batch_device(tok.handle, ids.data_ptr(), ids.numel(), rp.data_ptr(), None if rl is None else rl.data_ptr(),
                                                 n_rows, _lib.DECODE_SKIP_SPECIAL, stream, ctypes.byref(res)))
        call()
        nb = L.b2t_result_n_tokens(res)
        text = _device_view(torch, L.b2t_result_text(res), nb, torch.uint8, ids.device)
        toff = _device_view(torch, L.b2t_result_text_off(res), n_rows + 1, torch.int64, ids.device)
        check(text, toff)
        dev_text, dev_off = text.cpu().numpy(), toff.cpu().numpy().view(np.uint64)
        L.b2t_result_free(res)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(a.steps):
            call(); L.b2t_result_free(res)
        ev[1].record()
        torch.cuda.synchronize()
        t_dev = ev[0].elapsed_time(ev[1]) / 1e3 / a.steps
        L.b2t_engine_set_profiling(tok.handle, 1)
        call(); L.b2t_result_free(res)
        names = (ctypes.c_char_p * 16)(); ms = (ctypes.c_float * 16)()
        L.b2t_engine_last_kernels(tok.handle, names, ms, 16)
        kernels = {names[i].decode(): round(ms[i], 3) for i in range(16) if names[i] is not None}
        L.b2t_engine_set_profiling(tok.handle, 0)
        # host entry point: host ids in, pinned host text out
        h_ids = ids.cpu().numpy().view(np.uint32)
        h_rp = rp.cpu().numpy().view(np.uint64)
        h_rl = None if rl is None else rl.cpu().numpy().view(np.uint32)
        t0 = time.perf_counter()
        _lib.check(L.b2t_decode_batch(tok.handle, h_ids.ctypes.data, h_ids.size, h_rp.ctypes.data, None if h_rl is None else h_rl.ctypes.data, n_rows,
                                      _lib.DECODE_SKIP_SPECIAL, ctypes.byref(res)))
        t_host = time.perf_counter() - t0
        from tokenizers_b200.tokenizer import _view
        same = (np.array_equal(_view(L.b2t_result_text(res), L.b2t_result_n_tokens(res), np.uint8), dev_text) and
                np.array_equal(_view(L.b2t_result_text_off(res), n_rows + 1, np.uint64), dev_off))
        L.b2t_result_free(res)
        assert same, f"{name}: host and device entry points differ"
        # kernel time: the engine's records without the host's reads between them (*_read)
        kern_s = sum(v for kk, v in kernels.items() if not kk.endswith("_read")) / 1e3
        # tokens decoded: the rows' ids (with row lengths, the ids past a row's length are never read)
        n_tok = int(h_ids.size) if h_rl is None else int(h_rl.astype(np.int64).sum())
        moved = n_tok * 4 + (n_rows + 1) * 8 * (2 if rl is None else 1) + (0 if rl is None else n_rows * 4) + nb + (n_rows + 1) * 8
        w = {"rows": n_rows, "tokens": n_tok, "text_bytes": int(nb), "device_s": round(t_dev, 5), "host_s": round(t_host, 4),
             "device_tokens_per_s": round(n_tok / t_dev / 1e9, 3), "device_text_gb_s": round(nb / t_dev / 1e9, 2),
             "host_tokens_per_s": round(n_tok / t_host / 1e9, 3), "kernels_ms": kernels, "kernel_ms": round(kern_s * 1e3, 3),
             "roofline_share": round(moved / kern_s / (HBM_TBS * 1e12), 3) if kern_s else None, "rates_in": "G tokens/s, GB/s"}
        if wheel is not None:
            rows = []
            for r in range(min(a.wheel_docs, n_rows)):
                s = int(h_rp[r]); e = s + int(h_rl[r]) if h_rl is not None else int(h_rp[r + 1])
                rows.append(h_ids[s:e].tolist())
            ref = wheel.Tokenizer.from_str(tok._json)
            t0 = time.perf_counter()
            exp = ref.decode_batch(rows, skip_special_tokens=True)
            t_w = time.perf_counter() - t0
            ntok = sum(map(len, rows))
            got = [dev_text[int(dev_off[r]):int(dev_off[r + 1])].tobytes().decode("utf-8") for r in range(len(rows))]
            assert got == exp, f"{name}: differs from the reference wheel"
            w["wheel"] = {"rows": len(rows), "tokens": ntok, "threads": os.cpu_count(), "tokens_per_s": round(ntok / t_w / 1e6, 3), "rate_in": "M tokens/s",
                          "device_speedup": round((n_tok / t_dev) / (ntok / t_w), 1)}
        out["workloads"][name] = w
        log(f"{name}: {json.dumps(w)}")

    # (a) GPT-2 round trip
    tj = tokenizer("gpt2_style", {"type": "ByteLevel", "add_prefix_space": True, "trim_offsets": True, "use_regex": True})
    tok = Tokenizer.from_str(tj, device=0); tok._json = tj
    data, off, d_data, ids, rp = encode(tok, "gpt2")

    def check_a(text, toff):
        assert text.numel() == d_data.numel() and torch.equal(text, d_data), "the decoded text is not the corpus"
        assert np.array_equal(toff.cpu().numpy().view(np.uint64), off), "text offsets are not the document offsets"
    run("gpt2_roundtrip", tok, ids, rp, None, len(off) - 1, check_a)
    out["workloads"]["gpt2_roundtrip"]["byte_identical"] = True
    # (b) generation-like rows: [B, 2048] windows of the ids, random lengths
    W = 2048
    B = min(ids.numel() // W, 65536)
    g = torch.Generator(device="cpu").manual_seed(5)
    lens = torch.randint(1, W + 1, (B,), generator=g).to(torch.int32).cuda()
    rows_ids = ids[:B * W].contiguous()
    rpb = torch.arange(B, dtype=torch.int64, device=ids.device) * W
    run("gen_rows", tok, rows_ids, rpb, lens, B, lambda t, o: None)
    del ids, rp, rows_ids, d_data
    torch.cuda.empty_cache()
    # (c) WordPiece with cleanup
    tj = tokenizer("wordpiece", {"type": "WordPiece", "prefix": "##", "cleanup": True})
    tok = Tokenizer.from_str(tj, device=0); tok._json = tj
    data, off, d_data, ids, rp = encode(tok, "wordpiece")
    run("wordpiece", tok, ids, rp, None, len(off) - 1, lambda t, o: None)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
