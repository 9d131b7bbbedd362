"""Time HuggingFaceCrossEncoder.score on a ColBERT checkpoint next to two cross-encoders, in one run.

    python tools/bench_colbert.py [--calls 50] [--warmup 5] [--bulk-reps 3] [--json OUT]

Models: colbertv2.0 (BERT-base, dim 128, query_maxlen 32, doc_maxlen 180), the MiniLM-L6 cross-encoder
(ms-marco-MiniLM-L-6-v2) and bge-reranker-base, all ``synthetic:<preset>`` weights (timing does not depend on their
values).  RAGMeUp's call: one query of about 16 tokens against 14 documents of about 130 tokens; each call is timed on
the host clock and ends in its device synchronise (score returns host scores).  Bulk: one score call of 64 queries x
100 documents = 6 400 pairs, --bulk-reps times.  ColBERT encodes each distinct query and document once per call, a
cross-encoder every pair.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MODELS = ["synthetic:colbertv2.0:0", "synthetic:ms-marco-MiniLM-L-6-v2:0", "synthetic:bge-reranker-base:0"]


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")] if out else ("?", "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--bulk-reps", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the results here")
    a = ap.parse_args()
    import torch
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.tokenizer import synthetic_sentences, synthetic_vocab
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    vocab = synthetic_vocab(30522)
    queries = synthetic_sentences(vocab, a.calls + a.warmup, 15, 15, seed=1)
    docs = synthetic_sentences(vocab, 14, 120, 120, seed=2)
    bq = synthetic_sentences(vocab, 64, 15, 15, seed=3)
    bd = synthetic_sentences(vocab, 100, 120, 120, seed=4)
    bulk_pairs = [(q, d) for q in bq for d in bd]
    res = {"card": card(), "models": {}}
    for name in MODELS:
        ce = HuggingFaceCrossEncoder(model_name=name)
        for q in queries[:a.warmup]:
            ce.score([(q, d) for d in docs])
        ts = []
        for q in queries[a.warmup:]:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ce.score([(q, d) for d in docs])
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        ce.score(bulk_pairs)
        bulk = []
        for _ in range(a.bulk_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ce.score(bulk_pairs)
            torch.cuda.synchronize()
            bulk.append(time.perf_counter() - t0)
        res["models"][name] = {"call_ms_median": 1e3 * statistics.median(ts), "call_ms_min": 1e3 * min(ts),
                               "calls": len(ts), "bulk_6400_ms_median": 1e3 * statistics.median(bulk),
                               "bulk_pairs_per_s": 6400 / statistics.median(bulk)}
        print(json.dumps({name: res["models"][name]}), flush=True)
        del ce
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
