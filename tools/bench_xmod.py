"""Time ColBERT-XM (the colbert-xm preset: xmod-base, dim 128, query_maxlen 32, doc_maxlen 220) against the same
ColBERT without the language adapters (adapter_dim = 0, an XLM-R ColBERT of the same shape and weights), in one run.

    python tools/bench_xmod.py [--calls 50] [--warmup 5] [--bulk-reps 5] [--json OUT]

Two shapes: one query against 100 documents of about 150 tokens (a rerank call), and a bulk call of 64 queries x 100
documents = 6 400 pairs.  The two models alternate call by call, so drift on a shared host hits both alike.  Each call
is ColBERTScorer.score (host buffers in and out), timed on the host clock; it ends in its device synchronise.  The
adapter adds H^2 multiply-adds per token per layer to about 12 H^2 (+8 % GEMM work).  The card's name and power limit
are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from dataclasses import asdict

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")] if out else ("?", "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def texts(tok, n, words, seed):
    pieces = sorted(p[1:] for p in tok.get_vocab() if p.startswith("▁") and len(p) > 2)
    rng = np.random.default_rng(seed)
    return [" ".join(pieces[int(j)] for j in rng.integers(0, len(pieces), words)) for _ in range(n)]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--bulk-reps", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results here")
    a = ap.parse_args()
    import torch
    from ragmeup_b200.colbert import ColBERTScorer
    from ragmeup_b200.tokenizer import load_tokenizer
    from ragmeup_b200.weights import XLMRConfig, synthetic_colbert
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    cfg, w, lin, spec = synthetic_colbert("colbert-xm", 0)
    tok = load_tokenizer(None, cfg.vocab_size, xlmr=True)
    plain = XLMRConfig(**{k: v for k, v in asdict(cfg).items() if k not in ("adapter_dim", "languages", "language")})
    models = {"colbert-xm": ColBERTScorer(cfg, w, lin, spec, tok), "adapter_dim=0": ColBERTScorer(plain, w, lin, spec, tok)}
    qs = texts(tok, a.calls + a.warmup, 12, 1)
    docs = texts(tok, 100, 110, 2)
    bulk = [(q, d) for q in texts(tok, 64, 12, 3) for d in texts(tok, 100, 110, 4)]
    res = {"card": card(), "doc_tokens_mean": float(np.mean(np.diff(models["colbert-xm"].tokenizer.docs(docs)[1]))),
           "models": {}}
    call = {k: [] for k in models}
    for i, q in enumerate(qs):
        for name, m in models.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m.score([(q, d) for d in docs])
            torch.cuda.synchronize()
            if i >= a.warmup:
                call[name].append(time.perf_counter() - t0)
    for m in models.values():
        m.score(bulk)
    bt = {k: [] for k in models}
    for _ in range(a.bulk_reps):
        for name, m in models.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m.score(bulk)
            torch.cuda.synchronize()
            bt[name].append(time.perf_counter() - t0)
    for name in models:
        res["models"][name] = {"call_1x100_ms_median": 1e3 * statistics.median(call[name]),
                               "call_1x100_ms_min": 1e3 * min(call[name]), "calls": len(call[name]),
                               "bulk_64x100_ms_median": 1e3 * statistics.median(bt[name]),
                               "bulk_pairs_per_s": len(bulk) / statistics.median(bt[name])}
    x, p = res["models"]["colbert-xm"], res["models"]["adapter_dim=0"]
    res["adapter_cost"] = {"call": x["call_1x100_ms_median"] / p["call_1x100_ms_median"] - 1,
                           "bulk": x["bulk_64x100_ms_median"] / p["bulk_64x100_ms_median"] - 1}
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
