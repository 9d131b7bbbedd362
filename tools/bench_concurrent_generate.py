"""Time continuous batching (rmu_decoder_session_*) against sequential rmu_decoder_generate calls, in one run:

    python tools/bench_concurrent_generate.py [--layers 4] [--tokens 128] [--prompt 1024] [--reps 3] [--json OUT]

The workload is tools/bench_generate.py's: --layers synthetic layers of the Llama-3.1-8B shape (hidden 4 096, 32 / 8
heads, F 14 336, vocabulary 128 256), split planes and NF4 (two handles of the same weights), prompts of --prompt
random tokens, --tokens new tokens each, greedy, no eos.  For N = 1, 2, 4, 8 and 16 requests:
* sequential: N rmu_decoder_generate calls, one after another;
* together: the N requests join one session in one add, then steps until every row stops;
* staggered: one request joins every 16 steps (each add's prefill stalls the live rows; its time is reported).
The three run alternately --reps times; each figure is the median.  Aggregate tokens/s = N * tokens / wall time (the
prefills included).  The step time at each M is the median host time of session steps with M live rows (each step
ends in a stream synchronise).  The M = 1 session step is compared with rmu_decoder_generate's step, (a call of
1 + tokens - a one-token call) / tokens.  Every reply's tokens are checked against its solo run in the same process,
and the card's name and power limit are read in the same run.
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
from collections import defaultdict
from dataclasses import asdict, replace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

NS = (1, 2, 4, 8, 16)
STAGGER = 16


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")] if out else ("?", "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--prompt", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ns", default=",".join(map(str, NS)))
    ap.add_argument("--weights", default="split,nf4", help="the handles to time, split and / or nf4")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from ragmeup_b200 import _lib
    from ragmeup_b200.decode_session import DecodeSession, Request
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import DECODER_PRESETS, LlamaConfig, synthetic_llama_weights

    ns = [int(x) for x in args.ns.split(",")]
    cfg = replace(LlamaConfig(**asdict(DECODER_PRESETS["llama-3.1-8b"])), layers=args.layers, name="llama-3.1-8b")
    l = _lib.lib()
    w = synthetic_llama_weights(cfg, seed=0)
    lm = (0.02 * np.random.default_rng(1).standard_normal((cfg.vocab_size, cfg.hidden))).astype(np.float32)
    handles = {}
    for kind in args.weights.split(","):
        enc = BertEncoder(cfg, w, with_head=False)
        _lib.check(l.rmu_decoder_set_lm_head(enc._h, lm.ctypes.data), "rmu_decoder_set_lm_head")
        if kind == "nf4":
            _lib.check(l.rmu_decoder_quantize_nf4(enc._h, _lib.stream_ptr()), "rmu_decoder_quantize_nf4")
        handles[kind] = enc
    del lm, w
    s = _lib.SamplingC(0, 1.0, 1.0, 1.0, 50, 0, (C.c_int32 * _lib.MAX_EOS)())
    K, T = args.tokens, args.prompt
    rng = np.random.default_rng(0)
    prompts = [np.ascontiguousarray(rng.integers(0, cfg.vocab_size, T), dtype=np.int32) for _ in range(max(ns))]
    res = {"card": card(), "shape": "llama-3.1-8b", "layers": cfg.layers, "prompt": T, "tokens": K, "reps": args.reps,
           "rows": []}
    print(json.dumps(res["card"]), flush=True)

    for kind, enc in handles.items():
        out = np.zeros(K + 1, dtype=np.int32)
        n = C.c_int32(0)

        def generate(i, k=K):
            enc._check(l.rmu_decoder_generate(enc._h, prompts[i].ctypes.data, T, C.byref(s), i, k, out.ctypes.data,
                                              C.byref(n), None, _lib.stream_ptr()), "rmu_decoder_generate")
            return out[:n.value].tolist()

        solo = [generate(i) for i in range(max(ns))]              # also the warm-up of the single path
        sess = DecodeSession(enc)
        step_ms = defaultdict(list)                                # M -> session step times

        def sequential(N):
            t0 = time.perf_counter()
            got = [generate(i) for i in range(N)]
            torch.cuda.synchronize()
            assert got == solo[:N], "a sequential reply differs from its first run"
            return time.perf_counter() - t0, []

        def concurrent(N, stagger):
            toks = defaultdict(list)
            slot_of = {}
            adds = []

            def add(i):
                t0 = time.perf_counter()
                rows = sess.add([Request(prompts[i].tolist(), s, i, K)])
                adds.append((time.perf_counter() - t0) * 1e3)
                slot, tok, st = rows[0]
                assert st >= 0
                toks[i].append(tok)
                if st == _lib.GEN_LIVE:
                    slot_of[slot] = i

            t0 = time.perf_counter()
            if stagger:
                add(0)
            else:
                rows = sess.add([Request(prompts[i].tolist(), s, i, K) for i in range(N)])
                adds.append((time.perf_counter() - t0) * 1e3)
                for i, (slot, tok, st) in enumerate(rows):
                    toks[i].append(tok)
                    slot_of[slot] = i
            nxt, steps = 1 if stagger else N, 0
            while slot_of or nxt < N:
                if stagger and nxt < N and steps % STAGGER == 0 and steps > 0:
                    add(nxt)
                    nxt += 1
                if not slot_of:
                    steps += 1
                    continue
                M = len(slot_of)
                ts = time.perf_counter()
                rows = sess.step()
                step_ms[M].append((time.perf_counter() - ts) * 1e3)
                steps += 1
                for slot, tok, st in rows:
                    assert st >= 0
                    toks[slot_of[slot]].append(tok)
                    if st != _lib.GEN_LIVE:
                        del slot_of[slot]
            wall = time.perf_counter() - t0
            assert [toks[i] for i in range(N)] == solo[:N], "a session reply differs from its solo run"
            return wall, adds

        concurrent(2, False)                                      # warm-up: the session's cache and scratch
        for N in ns:
            walls = defaultdict(list)
            stalls = []
            for _ in range(args.reps):
                walls["sequential"].append(sequential(N)[0])
                walls["together"].append(concurrent(N, False)[0])
                w_st, adds = concurrent(N, True)
                walls["staggered"].append(w_st)
                stalls += adds[1:]
            row = {"weights": kind, "N": N}
            for mode, ws in walls.items():
                med = statistics.median(ws)
                row[f"{mode}_s"] = round(med, 4)
                row[f"{mode}_tok_s"] = round(N * K / med, 1)
            row["together_vs_sequential"] = round(row["together_tok_s"] / row["sequential_tok_s"], 3)
            row["staggered_vs_sequential"] = round(row["staggered_tok_s"] / row["sequential_tok_s"], 3)
            if stalls:
                row["staggered_add_ms_median"] = round(statistics.median(stalls), 3)
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
        # rmu_decoder_generate's step against the M = 1 session step
        ones, manys = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            generate(0, 1)
            torch.cuda.synchronize()
            ones.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            generate(0, K + 1)
            torch.cuda.synchronize()
            manys.append(time.perf_counter() - t0)
        gen_step = (statistics.median(manys) - statistics.median(ones)) / K * 1e3
        steps = {str(M): round(statistics.median(v), 3) for M, v in sorted(step_ms.items())}
        summary = {"weights": kind, "generate_step_ms": round(gen_step, 3), "session_step_ms_by_M": steps,
                   "session_M1_vs_generate": round(steps.get("1", float("nan")) / gen_step, 3)}
        res.setdefault("steps", []).append(summary)
        print(json.dumps(summary), flush=True)
        sess.close()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
