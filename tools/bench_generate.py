"""Time generation on the Llama-3.1-8B shape (hidden 4096, 32 / 8 heads, F 14336, vocabulary 128 256), in one run:

    python tools/bench_generate.py [--layers 4] [--tokens 32] [--weights split|nf4] [--json OUT]

For prompts of T = 1 024 and 4 096 tokens, greedy, with CUDA events around whole rmu_decoder_generate calls:
* prefill: a call that generates one token (the prefill, the LM head and the sampler);
* per decoded token: (a call of 1 + tokens - the one-token call) / tokens;
* the decode step split by the library's per-class timers: projections (E1 GEMMs without the LM head), decode
  attention with the KV cache writes, the LM head and the sampler (profiled in separate calls).
The synthetic model has --layers layers (all 32 are about 32 GB of host fp32); the per-layer parts are also scaled
to 32 layers, which is a COMPUTED extrapolation, not a measurement.  The floor it compares against is computed too:
30.0 GB of split-plane weights read once per token at 3.35 TB/s is at least 9.0 ms per token.  The card's name and
power limit are read in the same run.

With --weights nf4 the run holds two handles of the same weights, one split and one converted to NF4
(rmu_decoder_quantize_nf4), and alternates their calls; the NF4 decode step's projections are the "nf4" timer class.
It also times the decode GEMV alone on one layer's four projections of the full 8B shape (CUDA events over 200
launches of each) and states the share of 3.35 TB/s that their NF4 bytes (codes and absmax) reach.

    python tools/bench_generate.py --shape llama-3.1-70b [--layers 80] [--tokens 32] [--json OUT]

--shape llama-3.1-70b or qwen3-32b runs that shape in NF4 only, built layer by layer (BertEncoder.nf4_decoder) from
seeded per-layer weights drawn on the device with torch's generator (one seed per layer; no full-depth copy of the
model ever exists on the host), all layers by default.  It adds the load time (with the time spent drawing the
weights apart), the device bytes held after the load and after the LM head (cudaMemGetInfo, against
weights.decoder_memory_plan), and the GEMV's share of 3.35 TB/s on one layer of that shape.  The floor it states is
the NF4 layers plus the split-plane LM head read once per token.
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
from ragmeup_b200.weights import DecoderLayers  # noqa: E402

FULL_LAYERS = 32
PROF = {"gemm": 4, "decode_attention": 11, "lm_head": 12, "sampler": 13, "nf4": 14}
HBM_TBPS = 3.35


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


def gemv_share(cfg) -> dict:
    """the decode GEMV alone on one layer's q | k | v, o, gate | up and down at M = 1 (CUDA events, 200 launches each)"""
    import torch
    from ragmeup_b200 import _lib
    l = _lib.lib()
    H, F, QD, KD = cfg.hidden, cfg.ffn, cfg.heads * 128, cfg.kv_heads * 128
    shapes = {"qkv": (0, QD + 2 * KD, H), "o": (6, H, QD), "gate_up": (7, 2 * F, H), "down": (6, H, F)}
    out, total_ms, total_bytes = {}, 0.0, 0
    for name, (mode, N, K) in shapes.items():
        w = (torch.randn(N, K, device="cuda") * 0.02).half()
        codes = torch.empty(N * K // 2, dtype=torch.uint8, device="cuda")
        amax = torch.empty(N * K // 64, device="cuda")
        _lib.check(l.rmu_debug_nf4_quantize(w.data_ptr(), N * K, codes.data_ptr(), amax.data_ptr(), _lib.stream_ptr()))
        del w
        x = torch.randn(K, device="cuda").half()
        bias = torch.zeros(N, device="cuda")
        res = torch.zeros(N, device="cuda")
        half = torch.empty(N, dtype=torch.float16, device="cuda")

        def launch():
            _lib.check(l.rmu_debug_nf4_gemv(mode, x.data_ptr(), x.data_ptr(), codes.data_ptr(), amax.data_ptr(), N, K,
                                            bias.data_ptr(), res.data_ptr(), res.data_ptr(), half.data_ptr(),
                                            half.data_ptr(), None, _lib.stream_ptr()))
        for _ in range(20):
            launch()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(200):
            launch()
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / 200
        nbytes = N * K // 2 + N * K // 64 * 4
        out[name] = {"N": N, "K": K, "us": round(ms * 1e3, 2), "share_of_hbm_peak": round(nbytes / (ms * 1e-3) / (HBM_TBPS * 1e12), 3)}
        total_ms += ms
        total_bytes += nbytes
        del codes, amax
    out["layer"] = {"us": round(total_ms * 1e3, 2), "nf4_bytes": total_bytes,
                    "share_of_hbm_peak": round(total_bytes / (total_ms * 1e-3) / (HBM_TBPS * 1e12), 3)}
    return out


class SeededLayers(DecoderLayers):
    """seeded weights drawn on the device, one torch generator per tensor group: norms 1 + N(0, 0.1), embeddings and
    projections N(0, 0.02); ``draw_s`` sums the time spent drawing and copying to host"""

    def __init__(self, cfg, seed: int = 0):
        super().__init__(cfg)
        self.seed, self.draw_s = seed, 0.0

    def _draw(self, key: int, items):
        import torch
        t0 = time.perf_counter()
        g = torch.Generator(device="cuda").manual_seed(self.seed * 1_000_003 + key)
        out = {}
        for name, shape in items:
            a = torch.randn(shape, generator=g, device="cuda")
            a = 1.0 + 0.1 * a if name.endswith("norm.weight") or name.endswith("layernorm.weight") else 0.02 * a
            out[name] = a.cpu().numpy()
            del a
        torch.cuda.synchronize()
        self.draw_s += time.perf_counter() - t0
        return out

    def globals(self):
        c = self.cfg
        return self._draw(0, [("embed_tokens.weight", (c.vocab_size, c.hidden)), ("norm.weight", (c.hidden,))])

    def layer(self, l):
        return self._draw(1 + l, self.layer_names(l))


def large(args):
    """--shape llama-3.1-70b / qwen3-32b: the NF4 handle built layer by layer, then the same timings"""
    import torch
    from ragmeup_b200 import _lib
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import decoder_config, decoder_memory_plan
    cfg = replace(decoder_config("synthetic:" + args.shape), name=args.shape)
    if args.layers:
        cfg = replace(cfg, layers=args.layers)
    l = _lib.lib()
    res = {"card": card(), "shape": args.shape, "layers": cfg.layers, "weights": ["nf4"], "rows": []}
    print(json.dumps(res["card"]))
    plan = decoder_memory_plan(cfg, "nf4")
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    src = SeededLayers(cfg, seed=0)
    t0 = time.perf_counter()
    enc = BertEncoder.nf4_decoder(src)
    load_s = time.perf_counter() - t0
    torch.cuda.empty_cache()
    held = free0 - torch.cuda.mem_get_info()[0]
    lm = SeededLayers(cfg, seed=1)._draw(0, [("lm_head", (cfg.vocab_size, cfg.hidden))])["lm_head"]
    _lib.check(l.rmu_decoder_set_lm_head(enc._h, lm.ctypes.data), "rmu_decoder_set_lm_head")
    del lm
    torch.cuda.empty_cache()
    held_head = free0 - torch.cuda.mem_get_info()[0]
    res["load"] = {"load_s": round(load_s, 1), "of_which_drawing_weights_s": round(src.draw_s, 1),
                   "device_bytes_after_load": held, "planned_without_lm_head": plan["total"] - plan["lm_head"],
                   "device_bytes_with_lm_head": held_head, "planned_total": plan["total"],
                   "plan_gb": {k: round(v / 1e9, 3) for k, v in plan.items()}}
    print(json.dumps(res["load"]))
    nbytes = plan["layers"] + cfg.vocab_size * cfg.hidden * 4
    res["floor"] = {"bytes_per_token_computed": nbytes, "ms_per_token_at_3.35TBps_computed": round(nbytes / 3.35e9, 2)}
    print(json.dumps(res["floor"]))
    return cfg, {"nf4": enc}, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", choices=("llama-3.1-8b", "llama-3.1-70b", "qwen3-32b"), default="llama-3.1-8b")
    ap.add_argument("--layers", type=int, default=None)
    ap.add_argument("--tokens", type=int, default=32)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--weights", choices=("split", "nf4"), default="split")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from ragmeup_b200 import _lib
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import DECODER_PRESETS, LlamaConfig, synthetic_llama_weights

    l = _lib.lib()
    s = _lib.SamplingC(0, 1.0, 1.0, 1.0, 50, 0, (C.c_int32 * _lib.MAX_EOS)())
    if args.shape != "llama-3.1-8b":
        cfg, handles, res = large(args)
        full_layers = cfg.layers
    else:
        full_layers = FULL_LAYERS
        cfg = replace(LlamaConfig(**asdict(DECODER_PRESETS["llama-3.1-8b"])), layers=args.layers or 4,
                      name="llama-3.1-8b")
        w = synthetic_llama_weights(cfg, seed=0)
        lm = (0.02 * np.random.default_rng(1).standard_normal((cfg.vocab_size, cfg.hidden))).astype(np.float32)
        handles = {}
        for kind in (("split", "nf4") if args.weights == "nf4" else ("split",)):
            enc = BertEncoder(cfg, w, with_head=False)
            _lib.check(l.rmu_decoder_set_lm_head(enc._h, lm.ctypes.data), "rmu_decoder_set_lm_head")
            if kind == "nf4":
                _lib.check(l.rmu_decoder_quantize_nf4(enc._h, _lib.stream_ptr()), "rmu_decoder_quantize_nf4")
            handles[kind] = enc
        del lm, w
        res = {"card": card(), "shape": "llama-3.1-8b", "layers": cfg.layers, "weights": list(handles), "rows": []}
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

        def call(k, enc):
            t0 = time.perf_counter()
            enc._check(l.rmu_decoder_generate(enc._h, ids.ctypes.data, T, C.byref(s), 0, k, out.ctypes.data, C.byref(n),
                                              None, _lib.stream_ptr()), "rmu_decoder_generate")
            torch.cuda.synchronize()
            assert n.value == k
            return (time.perf_counter() - t0) * 1e3

        for enc in handles.values():
            call(args.tokens + 1, enc)                            # warm-up: cache and workspace growth, module load
        ones, manys = {k: [] for k in handles}, {k: [] for k in handles}
        for _ in range(args.calls):                               # the handles alternate call by call
            for kind, enc in handles.items():
                ones[kind].append(call(1, enc))
            for kind, enc in handles.items():
                manys[kind].append(call(args.tokens + 1, enc))
        for kind, enc in handles.items():
            one, many = statistics.median(ones[kind]), statistics.median(manys[kind])
            per_tok = (many - one) / args.tokens
            parts = {}
            for k in (1, args.tokens + 1):
                l.rmu_profile_reset()
                l.rmu_profile_enable(1)
                call(k, enc)
                l.rmu_profile_enable(0)
                for name, cls in PROF.items():
                    ms, cnt = C.c_double(), C.c_int64()
                    l.rmu_profile_read(cls, C.byref(ms), C.byref(cnt))
                    parts[name] = parts.get(name, 0.0) + (ms.value if k > 1 else -ms.value)
            step = {k: v / args.tokens for k, v in parts.items()}
            step["projections"] = step.pop("gemm") - step["lm_head"] + step.pop("nf4")
            scale = full_layers / cfg.layers
            row = {"weights": kind, "T": T, "prefill_ms": round(one, 3), "ms_per_token": round(per_tok, 3),
                   "step_ms": {k: round(v, 3) for k, v in step.items()}}
            if scale != 1:
                row[f"ms_per_token_{full_layers}_layers_extrapolated"] = round(
                    step["lm_head"] + step["sampler"] + scale * (per_tok - step["lm_head"] - step["sampler"]), 3)
            res["rows"].append(row)
            print(json.dumps(row))
    if "nf4" in handles:
        handles.clear()
        import gc
        gc.collect()
        res["nf4_gemv"] = gemv_share(cfg)
        print(json.dumps(res["nf4_gemv"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
