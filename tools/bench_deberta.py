"""Time the DeBERTa-v3 reranker mxbai-rerank-base-v1 next to bge-reranker-base (XLM-R) at equal shapes (768 hidden, 12
layers, 12 heads of 64), in one run.

    python tools/bench_deberta.py [--calls 50] [--warmup 5] [--bulk-reps 3] [--json OUT]

Two shapes: RAGMeUp's rerank call, one query against 14 documents of about 130 tokens per pair (85-word documents), and
a bulk call of 64 queries x 100 such documents = 6 400 pairs; the tokens per pair are reported.  The models alternate
call by call, so drift on a shared host hits both alike.  Each call is HuggingFaceCrossEncoder.score (host strings in, host scores out), timed on the host
clock; it ends in its device synchronise.  Then E2 ns per token and layer from the library's per-class CUDA-event
profile ("attention": for DeBERTa the two position-term launches and E2 with the terms, for bge E2 alone) over one bulk
call.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


DOC_WORDS = 85          # about 120 tokens of the synthetic Unigram vocabularies, so a pair is about 130


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
    ap.add_argument("--bulk-reps", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the results here")
    a = ap.parse_args()
    import torch
    from ragmeup_b200 import _lib
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    models = {"mxbai-rerank-base-v1": HuggingFaceCrossEncoder("synthetic:mxbai-rerank-base-v1"),
              "bge-reranker-base": HuggingFaceCrossEncoder("synthetic:bge-reranker-base")}
    work = {}
    for i, (name, m) in enumerate(models.items()):
        qs = texts(m.tokenizer, a.calls + a.warmup, 10, 1)
        docs = texts(m.tokenizer, 14, DOC_WORDS, 2)
        bulk = [(q, d) for q in texts(m.tokenizer, 64, 10, 3) for d in texts(m.tokenizer, 100, DOC_WORDS, 4)]
        ids, _typ, cu = m._pairs([q for q, _ in bulk], [d for _, d in bulk])
        work[name] = (qs, docs, bulk, int(cu[-1]))
    res = {"card": card(), "models": {}}
    call = {k: [] for k in models}
    for i in range(a.calls + a.warmup):
        for name, m in models.items():
            qs, docs, _, _ = work[name]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m.score([(qs[i], d) for d in docs])
            torch.cuda.synchronize()
            if i >= a.warmup:
                call[name].append(time.perf_counter() - t0)
    bt = {k: [] for k in models}
    for name, m in models.items():
        m.score(work[name][2])
    for _ in range(a.bulk_reps):
        for name, m in models.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m.score(work[name][2])
            torch.cuda.synchronize()
            bt[name].append(time.perf_counter() - t0)
    for name, m in models.items():
        qs, docs, bulk, bulk_tokens = work[name]
        _lib.profile_reset()
        _lib.profile_enable(True)
        m.score(bulk)
        torch.cuda.synchronize()
        prof = _lib.profile_read()
        _lib.profile_enable(False)
        ids, _typ, cu = m._pairs([qs[0]] * len(docs), docs)
        res["models"][name] = {
            "call_1x14_ms_median": 1e3 * statistics.median(call[name]), "call_1x14_ms_min": 1e3 * min(call[name]),
            "call_tokens_per_pair": float(np.mean(np.diff(cu))), "calls": len(call[name]),
            "bulk_64x100_ms_median": 1e3 * statistics.median(bt[name]),
            "bulk_pairs_per_s": len(bulk) / statistics.median(bt[name]), "bulk_tokens": bulk_tokens,
            "bulk_tokens_per_pair": bulk_tokens / len(bulk),
            "e2_ns_per_token_layer": 1e6 * prof["attention"][0] / (bulk_tokens * m.config.layers),
            "e2_launches": prof["attention"][1]}
    d, b = res["models"]["mxbai-rerank-base-v1"], res["models"]["bge-reranker-base"]
    res["deberta_over_bge"] = {"call": d["call_1x14_ms_median"] / b["call_1x14_ms_median"],
                               "bulk": d["bulk_64x100_ms_median"] / b["bulk_64x100_ms_median"],
                               "e2": d["e2_ns_per_token_layer"] / b["e2_ns_per_token_layer"]}
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
