"""Time attention provenance on the Llama-3.1-8B layer shape (hidden 4096, 32 / 8 heads, F 14336), in one run:

    python tools/bench_attention_provenance.py [--layers 2] [--calls 5] [--json OUT]

For each thread length T in {1 024, 4 096, 16 384}, with a chat-shaped span set (query, answer and ten documents
covering most of the thread), CUDA events time:
* the whole rmu_decoder_attention_spans call: L - 1 decoder layers, the last layer's attention inputs, the span kernels;
* the span kernels alone (A + B + C, rmu_debug_attention_spans) on planes of the same shape;
* per decoder layer, (call - span kernels) / (L - 1), which counts the last layer's partial step in with the others.
Beside the times it prints two COMPUTED byte counts (not measured): the library's activation workspace for the call,
and the L * heads * T^2 * 2 bytes that an eager transformers call with output_attentions=True holds for the
probabilities of L layers in fp16.  The default --layers 2 keeps the synthetic weights small (all 32 layers are about
32 GB of host fp32); pass --layers 32 for the whole model.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
from dataclasses import asdict, replace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")] if out else ("?", "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def chat_spans(T: int):
    """query, answer and ten documents: the documents fill 70% of the thread after a 5% system prompt"""
    doc0, dlen = T // 20, (7 * T // 10) // 10
    docs = [(doc0 + i * dlen, doc0 + (i + 1) * dlen - 1) for i in range(10)]
    q0 = doc0 + 10 * dlen + 8
    return [(q0, q0 + T // 50), (q0 + T // 50 + 8, T - 4)] + docs


def workspace_bytes(cfg, T: int) -> int:
    """the activation workspace of one call (rmu_encoder.cu: ensure_tokens_qwen3 and the span workspace)"""
    cap = (max(T, 1024) + 127) // 128 * 128
    QD, NQKV = cfg.heads * 128, (cfg.heads + 2 * cfg.kv_heads) * 128
    planes = 2 * 2 * cap * (cfg.hidden + QD + cfg.ffn + NQKV)
    fp32 = 4 * cap * (NQKV + cfg.hidden + 1)
    spans = 4 * cfg.heads * T * (2 + 32)
    return planes + fp32 + spans


def timed(torch, fn, calls):
    ms = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from ragmeup_b200 import _lib
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import DECODER_PRESETS, LlamaConfig, synthetic_llama_weights
    from oracle.encoder_kernels_ref import split_f16

    cfg = replace(LlamaConfig(**asdict(DECODER_PRESETS["llama-3.1-8b"])), layers=args.layers, name="llama-3.1-8b")
    enc = BertEncoder(cfg, synthetic_llama_weights(cfg, seed=0), with_head=False)
    l = _lib.lib()
    res = {"card": card(), "shape": "llama-3.1-8b", "layers": cfg.layers, "rows": []}
    print(json.dumps(res["card"]))
    rng = np.random.default_rng(0)
    for T in (1024, 4096, 16384):
        spans = chat_spans(T)
        ids = torch.from_numpy(rng.integers(0, cfg.vocab_size, T).astype(np.int32)).cuda()
        d_spans = torch.tensor(spans, dtype=torch.int32, device="cuda")
        out = torch.empty(len(spans), len(spans), dtype=torch.float64, device="cuda")
        NH = cfg.heads + 2 * cfg.kv_heads
        hi, lo = (torch.from_numpy(p).cuda() for p in split_f16(0.42 * rng.standard_normal((T, NH * 128))))

        def call():
            enc._check(l.rmu_decoder_attention_spans(enc._h, ids.data_ptr(), T, d_spans.data_ptr(), len(spans),
                                                     out.data_ptr(), _lib.stream_ptr()), "rmu_decoder_attention_spans")

        def kernels():
            _lib.check(l.rmu_debug_attention_spans(hi.data_ptr(), lo.data_ptr(), T, cfg.heads, cfg.kv_heads,
                                                   d_spans.data_ptr(), len(spans), out.data_ptr(), C.c_void_p(
                                                       _lib.stream_ptr())), "rmu_debug_attention_spans")

        call(), kernels()                                        # warm-up: workspace growth, module load
        t_call, t_spans = timed(torch, call, args.calls), timed(torch, kernels, args.calls)
        row = {"T": T, "call_ms": round(t_call, 3), "span_kernels_ms": round(t_spans, 3),
               "per_layer_ms": round((t_call - t_spans) / max(1, cfg.layers - 1), 3),
               "workspace_bytes_computed": workspace_bytes(cfg, T),
               "reference_eager_attention_bytes_computed_32_layers": 32 * cfg.heads * T * T * 2}
        res["rows"].append(row)
        print(json.dumps(row))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
