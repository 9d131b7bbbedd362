"""Time LLM provenance's generation on the Llama-3.1-8B shape (hidden 4096, 32 / 8 heads, F 14336, vocabulary 128 256):
B scoring prompts that share P tokens and have S = 200 tokens each of their own, 10 new tokens each (greedy, no eos,
so every row runs all 10 steps), in one run:

    python tools/bench_llm_provenance.py [--layers 4] [--calls 3] [--json OUT]

For B in {3, 10} and P in {512, 1024}, on a split handle and an NF4 handle of the same synthetic weights, it alternates
B sequential rmu_decoder_generate calls with one rmu_decoder_generate_batch call (host clock around each, after a
device synchronise), checks that both give the same tokens, and reports the median of --calls pairs.  It also times
the multi-row NF4 GEMV alone (rmu_debug_nf4_gemv_rows, CUDA events over 100 launches) on one full-shape layer's four
projections at M = 1, 4, 10 and 16, as a share of 3.35 TB/s for the layer's NF4 bytes (codes and absmax, read once
per launch whatever M is).  The 32-layer figures scale the per-layer part of the --layers run: a COMPUTED
extrapolation, not a measurement.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time
from dataclasses import asdict, replace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_generate import HBM_TBPS, card  # noqa: E402

S, NEW = 200, 10


def gemv_rows_share(cfg) -> dict:
    import torch
    from ragmeup_b200 import _lib
    l = _lib.lib()
    H, F, QD, KD = cfg.hidden, cfg.ffn, cfg.heads * 128, cfg.kv_heads * 128
    shapes = {"qkv": (0, QD + 2 * KD, H), "o": (6, H, QD), "gate_up": (7, 2 * F, H), "down": (6, H, F)}
    weights = {}
    for name, (mode, N, K) in shapes.items():
        w = (torch.randn(N, K, device="cuda") * 0.02).half()
        codes = torch.empty(N * K // 2, dtype=torch.uint8, device="cuda")
        amax = torch.empty(N * K // 64, device="cuda")
        _lib.check(l.rmu_debug_nf4_quantize(w.data_ptr(), N * K, codes.data_ptr(), amax.data_ptr(), _lib.stream_ptr()))
        weights[name] = (mode, N, K, codes, amax)
        del w
    out = {}
    for M in (1, 4, 10, 16):
        total_ms, total_bytes = 0.0, 0
        for name, (mode, N, K, codes, amax) in weights.items():
            x = torch.randn(M, K, device="cuda").half()
            bias = torch.zeros(N, device="cuda")
            res = torch.zeros(M, N, device="cuda")
            half = torch.empty(M, N, dtype=torch.float16, device="cuda")

            def launch():
                _lib.check(l.rmu_debug_nf4_gemv_rows(mode, M, x.data_ptr(), x.data_ptr(), codes.data_ptr(),
                                                     amax.data_ptr(), N, K, bias.data_ptr(), res.data_ptr(),
                                                     res.data_ptr(), half.data_ptr(), half.data_ptr(), None,
                                                     _lib.stream_ptr()))
            for _ in range(10):
                launch()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(100):
                launch()
            b.record()
            torch.cuda.synchronize()
            total_ms += a.elapsed_time(b) / 100
            total_bytes += N * K // 2 + N * K // 64 * 4
        out[f"M={M}"] = {"layer_us": round(total_ms * 1e3, 1),
                         "share_of_hbm_peak": round(total_bytes / (total_ms * 1e-3) / (HBM_TBPS * 1e12), 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from ragmeup_b200 import _lib
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import DECODER_PRESETS, LlamaConfig, synthetic_llama_weights

    cfg = replace(LlamaConfig(**asdict(DECODER_PRESETS["llama-3.1-8b"])), layers=args.layers, name="llama-3.1-8b")
    l = _lib.lib()
    res = {"card": card(), "shape": "llama-3.1-8b", "layers": cfg.layers, "S": S, "new_tokens": NEW, "rows": []}
    print(json.dumps(res["card"]), flush=True)
    res["gemv_rows"] = gemv_rows_share(cfg)
    print(json.dumps(res["gemv_rows"]), flush=True)
    w = synthetic_llama_weights(cfg, seed=0)
    lm = (0.02 * np.random.default_rng(1).standard_normal((cfg.vocab_size, cfg.hidden))).astype(np.float32)
    handles = {}
    for kind in ("split", "nf4"):
        enc = BertEncoder(cfg, w, with_head=False)
        _lib.check(l.rmu_decoder_set_lm_head(enc._h, lm.ctypes.data), "rmu_decoder_set_lm_head")
        if kind == "nf4":
            _lib.check(l.rmu_decoder_quantize_nf4(enc._h, _lib.stream_ptr()), "rmu_decoder_quantize_nf4")
        handles[kind] = enc
    del lm, w
    s = _lib.SamplingC(0, 1.0, 1.0, 1.0, 50, 0, (C.c_int32 * _lib.MAX_EOS)())
    rng = np.random.default_rng(0)
    for P in (512, 1024):
        prefix = rng.integers(0, cfg.vocab_size, P).tolist()
        for B in (3, 10):
            prompts = [prefix + rng.integers(0, cfg.vocab_size, S).tolist() for _ in range(B)]
            ids = np.ascontiguousarray([t for p in prompts for t in p], dtype=np.int32)
            cu = np.ascontiguousarray(np.cumsum([0] + [len(p) for p in prompts]), dtype=np.int32)
            seeds = np.zeros(B, dtype=np.uint64)
            for kind, enc in handles.items():
                def sequential():
                    toks = []
                    for p in prompts:
                        a = np.ascontiguousarray(p, dtype=np.int32)
                        out, n = np.zeros(NEW, dtype=np.int32), C.c_int32(0)
                        _lib.check(l.rmu_decoder_generate(enc._h, a.ctypes.data, len(p), C.byref(s), 0, NEW,
                                                          out.ctypes.data, C.byref(n), None, _lib.stream_ptr()))
                        toks.append(out[:n.value].tolist())
                    return toks

                def batch():
                    out, n = np.zeros((B, NEW), dtype=np.int32), np.zeros(B, dtype=np.int32)
                    _lib.check(l.rmu_decoder_generate_batch(enc._h, ids.ctypes.data, cu.ctypes.data, B, C.byref(s),
                                                            seeds.ctypes.data, NEW, out.ctypes.data, n.ctypes.data,
                                                            None, _lib.stream_ptr()))
                    return [out[b, :n[b]].tolist() for b in range(B)]

                def timed(f):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    r = f()
                    torch.cuda.synchronize()
                    return (time.perf_counter() - t0) * 1e3, r

                sequential(), batch()                           # warm-up: cache and workspaces at this shape
                ts, tb, equal = [], [], True
                for _ in range(args.calls):
                    a, ra = timed(sequential)
                    b, rb = timed(batch)
                    ts.append(a)
                    tb.append(b)
                    equal &= ra == rb and all(len(r) == NEW for r in rb)
                ms_s, ms_b = statistics.median(ts), statistics.median(tb)
                row = {"weights": kind, "B": B, "P": P, "sequential_ms": round(ms_s, 2), "batch_ms": round(ms_b, 2),
                       "speedup": round(ms_s / ms_b, 2), "tokens_equal": bool(equal)}
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
                if not equal:
                    raise SystemExit("batched and sequential tokens differ")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
