"""Time FlashrankRerank.compress_documents at RAGMeUp's rerank call shape on each FlashRank BERT shape.

    python tools/bench_flashrank.py [--calls 50] [--warmup 5] [--bulk-reps 3] [--json OUT]

The call shape: one query of about 16 tokens against 14 documents of about 130 tokens (vector_store_k = 10 MMR
results plus BM25's 4, before de-duplication).  Each shape is warmed up, then --calls calls are timed one by one on
the host clock, each ending in its device synchronise (the call returns host scores, so the device work is done when
it returns).  The median and minimum are reported.  The bulk case is 64 queries x 100 documents: 64 calls back to
back, --bulk-reps times.  Weights are synthetic (``synthetic:<preset>``); timing does not depend on their values.  The
card's name and power limit are read in the same run.  There is no CPU FlashRank arm: flashrank and onnxruntime are
not part of this project's environment, so no CPU time is reported.
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

SHAPES = ["ms-marco-MultiBERT-L-12", "ms-marco-TinyBERT-L-2-v2", "ms-marco-MiniLM-L-12-v2"]


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
    from ragmeup_b200.documents import Document
    from ragmeup_b200.flashrank import FlashrankRerank
    from ragmeup_b200.tokenizer import synthetic_sentences, synthetic_vocab
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    res = {"card": card(), "shapes": {}}
    for preset in SHAPES:
        fr = FlashrankRerank(model=f"synthetic:{preset}:0:4.0", top_n=3)
        vocab = synthetic_vocab(fr.client.config.vocab_size)
        queries = synthetic_sentences(vocab, a.calls + a.warmup, 15, 15, seed=1)
        docs = [Document(t, {}) for t in synthetic_sentences(vocab, 14, 128, 128, seed=2)]
        _, _, cu = fr.client._pairs([queries[0]] * 14, [d.page_content for d in docs])
        tok = np.diff(cu)
        for q in queries[:a.warmup]:
            fr.compress_documents(docs, q)
        ts = []
        for q in queries[a.warmup:]:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fr.compress_documents(docs, q)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        # bulk: 64 queries x 100 documents; after the warm-up call the documents' WordPiece ids are cached, as in a
        # server that reranks the same chunks for many queries
        bq = synthetic_sentences(vocab, 64, 15, 15, seed=3)
        bd = [Document(t, {}) for t in synthetic_sentences(vocab, 100, 128, 128, seed=4)]
        fr.compress_documents(bd, bq[0])
        bulk = []
        for _ in range(a.bulk_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for q in bq:
                fr.compress_documents(bd, q)
            torch.cuda.synchronize()
            bulk.append(time.perf_counter() - t0)
        res["shapes"][preset] = {
            "pair_tokens_mean": float(tok.mean()), "pair_tokens_max": int(tok.max()),
            "call_ms_median": 1e3 * statistics.median(ts), "call_ms_min": 1e3 * min(ts), "calls": len(ts),
            "bulk_64x100_ms_median": 1e3 * statistics.median(bulk), "bulk_64x100_ms_min": 1e3 * min(bulk),
            "bulk_pairs_per_s": 6400 / statistics.median(bulk),
        }
        print(json.dumps({preset: res["shapes"][preset]}), flush=True)
        del fr
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
