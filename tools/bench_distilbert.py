"""Time distiluse-base-multilingual-cased-v2 (DistilBERT + a sentence-transformers Dense 768 -> 512 tanh) against the same
encoder without its Dense module, and the Dense kernel alone.

    python tools/bench_distilbert.py [--calls 200] [--warmup 20] [--bulk-reps 5] [--dense-reps 200] [--json OUT]

* query: ``embed_query`` on one text of about 16 tokens (RAGMeUp's query shape), --calls calls timed one by one on the
  host clock; each returns host floats, so the device work is done when it returns.  Median and minimum.
* ingest: ``embed_documents`` on 1 000 chunks of about 128 tokens (RAGMeUp's ingest shape), --bulk-reps times.
* models: ``synthetic:distiluse-base-multilingual-cased-v2`` as it loads (mean pooling, Dense, 512 wide), and the same
  weights without the Dense module (768 wide); the two are timed alternately, call by call.
* dense: ``rmu_debug_dense`` (768 -> 512, tanh, bias) on 1 000 pooled rows, CUDA events around --dense-reps launches.

Weights are synthetic; timing does not depend on their values.  The card's name and power limit are read in the same
run.
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
NAME = "synthetic:distiluse-base-multilingual-cased-v2"


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")] if out else ("?", "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def models():
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import resolve_model
    dense = HuggingFaceEmbeddings(model_name=NAME)
    plain = HuggingFaceEmbeddings(model_name=NAME)
    cfg, w, *_ = resolve_model(NAME, with_head=False)
    plain.client = BertEncoder(cfg, {k: v for k, v in w.items() if not k.startswith("dense.")}, with_head=False)
    return {"distiluse with Dense": dense, "distiluse without Dense": plain}


def time_models(embs, a) -> dict:
    import torch
    from ragmeup_b200.tokenizer import synthetic_sentences
    first = next(iter(embs.values()))
    vocab = first.tokenizer.get_vocab()
    queries = synthetic_sentences(vocab, a.calls + a.warmup, 14, 14, seed=1)
    docs = synthetic_sentences(vocab, 1000, 126, 126, seed=2)
    res = {k: {"query": [], "ingest": []} for k in embs}
    for emb in embs.values():
        for q in queries[:a.warmup]:
            emb.embed_query(q)
        emb.embed_documents(docs)
    for q in queries[a.warmup:]:
        for k, emb in embs.items():
            t0 = time.perf_counter()
            emb.embed_query(q)
            res[k]["query"].append(time.perf_counter() - t0)
    for _ in range(a.bulk_reps):
        for k, emb in embs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            emb.embed_documents(docs)
            res[k]["ingest"].append(time.perf_counter() - t0)
    out = {}
    for k, emb in embs.items():
        q, b = res[k]["query"], res[k]["ingest"]
        out[k] = {"width": emb.client.embed_dim,
                  "query_tokens_mean": float(np.mean(np.diff(emb._ragged(queries[:50])[2]))),
                  "chunk_tokens_mean": float(np.mean(np.diff(emb._ragged(docs)[2]))),
                  "query_ms_median": 1e3 * statistics.median(q), "query_ms_min": 1e3 * min(q),
                  "ingest_1000_ms_median": 1e3 * statistics.median(b), "ingest_1000_ms_min": 1e3 * min(b)}
    return out


def time_dense(a) -> dict:
    import torch
    from ragmeup_b200 import _lib
    B, n_in, n_out = 1000, 768, 512
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, n_in, device="cuda", generator=g)
    W = torch.randn(n_out, n_in, device="cuda", generator=g) / n_in ** 0.5
    b = torch.randn(n_out, device="cuda", generator=g)
    y = torch.empty(B, n_out, device="cuda")
    st = _lib.stream_ptr()

    def run():
        _lib.check(_lib.lib().rmu_debug_dense(x.data_ptr(), B, n_in, n_out, W.data_ptr(), b.data_ptr(), 1, 0,
                                              y.data_ptr(), st))
    for _ in range(10):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.dense_reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / a.dense_reps
    return {"rows": B, "in": n_in, "out": n_out, "us_per_launch": us, "gflop": 2e-9 * B * n_in * n_out,
            "gflop_per_s": 2e-9 * B * n_in * n_out / (us * 1e-6)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--bulk-reps", type=int, default=5)
    ap.add_argument("--dense-reps", type=int, default=200)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = {"card": card(), "models": time_models(models(), a), "dense_kernel": time_dense(a)}
    print(json.dumps(res, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
