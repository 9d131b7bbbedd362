"""Time generation on the Llama-3.1-8B shape (hidden 4096, 32 / 8 heads, F 14336, vocabulary 128 256), in one run:

    python tools/bench_generate.py [--layers 4] [--tokens 32] [--json OUT]

For prompts of T = 1 024 and 4 096 tokens, greedy, with CUDA events around whole rmu_decoder_generate calls:
* prefill: a call that generates one token (the prefill, the LM head and the sampler);
* per decoded token: (a call of 1 + tokens - the one-token call) / tokens;
* the decode step split by the library's per-class timers: projections (E1 GEMMs without the LM head), decode
  attention with the KV cache writes, the LM head and the sampler (profiled in separate calls).
The synthetic model has --layers layers (all 32 are about 32 GB of host fp32); the per-layer parts are also scaled
to 32 layers, which is a COMPUTED extrapolation, not a measurement.  The floor it compares against is computed too:
30.0 GB of split-plane weights read once per token at 3.35 TB/s is at least 9.0 ms per token.  The card's name and
power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time
from dataclasses import asdict, replace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FULL_LAYERS = 32
PROF = {"gemm": 4, "decode_attention": 11, "lm_head": 12, "sampler": 13}


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")] if out else ("?", "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def split_plane_bytes(cfg, layers: int) -> int:
    """the weights one decode step reads: per layer q | k | v, o, gate | up, down, plus the LM head, two fp16 planes"""
    H, F, QD, KD = cfg.hidden, cfg.ffn, cfg.heads * 128, cfg.kv_heads * 128
    per_layer = H * (QD + 2 * KD) + QD * H + 2 * F * H + F * H
    return 4 * (layers * per_layer + cfg.vocab_size * H)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--tokens", type=int, default=32)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from ragmeup_b200 import _lib
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import DECODER_PRESETS, LlamaConfig, synthetic_llama_weights

    cfg = replace(LlamaConfig(**asdict(DECODER_PRESETS["llama-3.1-8b"])), layers=args.layers, name="llama-3.1-8b")
    enc = BertEncoder(cfg, synthetic_llama_weights(cfg, seed=0), with_head=False)
    l = _lib.lib()
    lm = (0.02 * np.random.default_rng(1).standard_normal((cfg.vocab_size, cfg.hidden))).astype(np.float32)
    _lib.check(l.rmu_decoder_set_lm_head(enc._h, lm.ctypes.data), "rmu_decoder_set_lm_head")
    del lm
    s = _lib.SamplingC(0, 1.0, 1.0, 1.0, 50, 0, (C.c_int32 * _lib.MAX_EOS)())
    res = {"card": card(), "shape": "llama-3.1-8b", "layers": cfg.layers, "rows": []}
    print(json.dumps(res["card"]))
    full_gb = split_plane_bytes(cfg, FULL_LAYERS) / 1e9
    res["floor"] = {"split_plane_gb_32_layers_computed": round(full_gb, 2),
                    "ms_per_token_at_3.35TBps_computed": round(full_gb / 3.35, 2)}
    print(json.dumps(res["floor"]))
    rng = np.random.default_rng(0)
    for T in (1024, 4096):
        ids = np.ascontiguousarray(rng.integers(0, cfg.vocab_size, T), dtype=np.int32)
        out = np.zeros(args.tokens + 1, dtype=np.int32)
        n = C.c_int32(0)

        def call(k):
            t0 = time.perf_counter()
            enc._check(l.rmu_decoder_generate(enc._h, ids.ctypes.data, T, C.byref(s), 0, k, out.ctypes.data, C.byref(n),
                                              None, _lib.stream_ptr()), "rmu_decoder_generate")
            torch.cuda.synchronize()
            assert n.value == k
            return (time.perf_counter() - t0) * 1e3

        call(args.tokens + 1)                                     # warm-up: cache and workspace growth, module load
        one = statistics.median(call(1) for _ in range(args.calls))
        many = statistics.median(call(args.tokens + 1) for _ in range(args.calls))
        per_tok = (many - one) / args.tokens
        parts = {}
        for k in (1, args.tokens + 1):
            l.rmu_profile_reset()
            l.rmu_profile_enable(1)
            call(k)
            l.rmu_profile_enable(0)
            for name, cls in PROF.items():
                ms, cnt = C.c_double(), C.c_int64()
                l.rmu_profile_read(cls, C.byref(ms), C.byref(cnt))
                parts[name] = parts.get(name, 0.0) + (ms.value if k > 1 else -ms.value)
        step = {k: v / args.tokens for k, v in parts.items()}
        step["projections"] = step.pop("gemm") - step["lm_head"]
        scale = FULL_LAYERS / cfg.layers
        row = {"T": T, "prefill_ms": round(one, 3), "ms_per_token": round(per_tok, 3),
               "step_ms": {k: round(v, 3) for k, v in step.items()},
               "ms_per_token_32_layers_extrapolated": round(step["lm_head"] + step["sampler"] +
                                                            scale * (per_tok - step["lm_head"] - step["sampler"]), 3)}
        res["rows"].append(row)
        print(json.dumps(row))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
