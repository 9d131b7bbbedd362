"""Time prompt-lookup decoding on the Llama-3.1-8B shape (hidden 4096, 32 / 8 heads, F 14336, vocabulary 128 256), in
one run:
    python tools/bench_prompt_lookup.py [--layers 4] [--calls 3] [--json OUT]
The run holds two handles of the same synthetic weights, one on split planes and one converted to NF4, and alternates
their calls.  For prompts of T = 1 024 and 4 096 tokens, greedy, every time a median of --calls whole calls timed with
the host clock (each call ends in a synchronise):
1. pass cost against k = 0, 1, 3, 7, 15: a call of 65 new tokens whose injected drafts (rmu_debug_generate_drafts) are
   all accepted, less a one-token call (the prefill), over its passes -> ms per pass and tokens per pass.  k = 0 is
   rmu_decoder_generate.
2. whole calls of 128 new tokens: rmu_decoder_generate against injected drafts at k = 7 that are all rejected (every
   draft wrong: the overhead case), half wrong (every other draft) and all accepted -> tokens/s and passes; every call
   returns the plain call's tokens (asserted).
The synthetic weights say nothing about how often real RAGMeUp answers accept drafts: the acceptance here is set by
the injected drafts.  The card's name and power limit are read in the same run.
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

KS = (0, 1, 3, 7, 15)
PASS_TOKENS = 65
CALL_TOKENS = 128


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")] if out else ("?", "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from ragmeup_b200 import _lib
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import DECODER_PRESETS, LlamaConfig, synthetic_llama_weights
    cfg = replace(LlamaConfig(**asdict(DECODER_PRESETS["llama-3.1-8b"])), layers=args.layers, name="llama-3.1-8b")
    l = _lib.lib()
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
    V = cfg.vocab_size
    res = {"card": card(), "shape": "llama-3.1-8b", "layers": cfg.layers, "calls": args.calls, "pass_cost": [],
           "whole_calls": []}
    print(json.dumps(res["card"]), flush=True)

    def run(enc, ids, max_new, k=None, drafts=None):
        """(seconds, tokens, passes): rmu_decoder_generate when k is None, else rmu_debug_generate_drafts"""
        out = np.zeros(max_new, dtype=np.int32)
        n, passes = C.c_int32(0), C.c_int32(0)
        t0 = time.perf_counter()
        if k is None:
            rc = l.rmu_decoder_generate(enc._h, ids.ctypes.data, len(ids), C.byref(s), 0, max_new, out.ctypes.data,
                                        C.byref(n), None, _lib.stream_ptr())
            passes.value = n.value - 1
        else:
            d = np.ascontiguousarray(drafts, dtype=np.int32)
            rc = l.rmu_debug_generate_drafts(enc._h, ids.ctypes.data, len(ids), C.byref(s), 0, max_new, d.ctypes.data,
                                             k, out.ctypes.data, C.byref(n), None, C.byref(passes), _lib.stream_ptr())
        dt = time.perf_counter() - t0
        enc._check(rc, "generate")
        return dt, out[:n.value].tolist(), passes.value

    rng = np.random.default_rng(0)
    for T in (1024, 4096):
        ids = np.ascontiguousarray(rng.integers(0, V, T), dtype=np.int32)
        plain = {kind: run(enc, ids, CALL_TOKENS)[1] for kind, enc in handles.items()}      # warm-up and the drafts
        for kind in handles:
            assert len(plain[kind]) == CALL_TOKENS

        def wrong_every(toks, j):
            return [(t + 1) % V if m % j == 0 else t for m, t in enumerate(toks)]

        # 1. pass cost against k, every draft accepted
        for k in KS:
            times = {kind: [] for kind in handles}
            for _ in range(args.calls):
                for kind, enc in handles.items():
                    toks = plain[kind][:PASS_TOKENS]
                    t1 = run(enc, ids, 1)[0]
                    dt, got, passes = run(enc, ids, PASS_TOKENS) if k == 0 else run(enc, ids, PASS_TOKENS, k, toks)
                    assert got == toks
                    times[kind].append(((dt - t1) / passes, passes))
            for kind in handles:
                ms = statistics.median(t for t, _ in times[kind]) * 1e3
                passes = times[kind][0][1]
                row = {"T": T, "weights": kind, "k": k, "passes": passes,
                       "tokens_per_pass": round((PASS_TOKENS - 1) / passes, 2), "ms_per_pass": round(ms, 3)}
                res["pass_cost"].append(row)
                print(json.dumps(row), flush=True)
        # 2. whole calls of 128 tokens at k = 7
        variants = {"plain": None, "accept_0": lambda t: wrong_every(t, 1), "accept_50": lambda t: wrong_every(t, 2),
                    "accept_100": lambda t: list(t)}
        for name, make in variants.items():
            times = {kind: [] for kind in handles}
            for _ in range(args.calls):
                for kind, enc in handles.items():
                    if make is None:
                        dt, got, passes = run(enc, ids, CALL_TOKENS)
                    else:
                        dt, got, passes = run(enc, ids, CALL_TOKENS, 7, make(plain[kind]))
                    assert got == plain[kind], (name, kind)
                    times[kind].append((dt, passes))
            for kind in handles:
                dt = statistics.median(t for t, _ in times[kind])
                row = {"T": T, "weights": kind, "drafts": name, "k": 0 if make is None else 7,
                       "passes": times[kind][0][1], "tokens_per_s": round(CALL_TOKENS / dt, 1),
                       "call_ms": round(dt * 1e3, 1)}
                res["whole_calls"].append(row)
                print(json.dumps(row), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
