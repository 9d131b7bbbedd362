"""Time MPNet sentence embeddings against a BERT encoder of the same shape and pooling, and E2 attention with and
without MPNet's relative position bias.

    python tools/bench_mpnet.py [--calls 200] [--warmup 20] [--bulk-reps 5] [--att-reps 50] [--json OUT]

* query: ``embed_query`` on one text of about 16 tokens (RAGMeUp's query shape), --calls calls timed one by one on the
  host clock; each returns host floats, so the device work is done when it returns.  Median and minimum.
* ingest: ``embed_documents`` on 1 000 chunks of about 128 tokens (RAGMeUp's ingest shape), --bulk-reps times.
* models: ``synthetic:all-mpnet-base-v2`` (768 / 12 layers / 12 heads / 3072, mean pooling, Normalize, 384 tokens) and
  the BERT of the same shape, ``synthetic:bge-base-en-v1.5`` switched to mean pooling, Normalize and 384 tokens.  The
  two use different synthetic vocabularies, so their token counts are reported next to the times.
* attention: ``rmu_debug_attention`` and ``rmu_debug_attention_bias`` (10 warps, the encoder's configuration) on the
  same QKV planes of the ingest batch (12 heads, d_h 64), CUDA events around --att-reps launches of each, alternated.

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


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")] if out else ("?", "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def models():
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.tokenizer import RaggedTokenizer
    mp = HuggingFaceEmbeddings(model_name="synthetic:all-mpnet-base-v2")
    bert = HuggingFaceEmbeddings(model_name="synthetic:bge-base-en-v1.5")
    bert.pooling, bert.normalize, bert.max_seq_length = "mean", True, 384
    bert._ragged = RaggedTokenizer(bert.tokenizer, 384)
    return {"mpnet all-mpnet-base-v2": mp, "bert 768/12 mean": bert}


def time_model(emb, a) -> dict:
    import torch
    from ragmeup_b200.tokenizer import synthetic_sentences
    vocab = emb.tokenizer.get_vocab()
    queries = synthetic_sentences(vocab, a.calls + a.warmup, 14, 14, seed=1)
    docs = synthetic_sentences(vocab, 1000, 126, 126, seed=2)
    q_tok = float(np.mean(np.diff(emb._ragged(queries[:50])[2])))
    d_tok = float(np.mean(np.diff(emb._ragged(docs)[2])))
    for q in queries[:a.warmup]:
        emb.embed_query(q)
    ts = []
    for q in queries[a.warmup:]:
        t0 = time.perf_counter()
        emb.embed_query(q)
        ts.append(time.perf_counter() - t0)
    emb.embed_documents(docs)
    bulk = []
    for _ in range(a.bulk_reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        emb.embed_documents(docs)
        bulk.append(time.perf_counter() - t0)
    return {"query_tokens_mean": q_tok, "query_ms_median": 1e3 * statistics.median(ts), "query_ms_min": 1e3 * min(ts),
            "chunk_tokens_mean": d_tok, "ingest_1000_ms_median": 1e3 * statistics.median(bulk),
            "ingest_1000_ms_min": 1e3 * min(bulk), "ingest_chunks_per_s": 1000 / statistics.median(bulk)}


def time_attention(a, cu) -> dict:
    """E2 with and without the bias on the same planes; ms per launch (all sequences, all heads)"""
    import torch
    from ragmeup_b200 import _lib
    H, heads = 768, 12
    T = int(cu[-1])
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(T, 3 * H, device="cuda", generator=g)
    qkv[:, :H] *= 1.4426950408889634 / 8.0
    hi = qkv.half()
    lo = (qkv - hi.float()).half()
    bias = np.random.default_rng(0).standard_normal((32, heads)).astype(np.float32)
    tab = np.zeros((heads, 255), np.float32)
    _lib.check(_lib.lib().rmu_relative_bias_table(bias.ctypes.data, 32, heads, tab.ctypes.data))
    tab = torch.from_numpy(tab).cuda()
    cu_d = torch.from_numpy(np.asarray(cu, np.int32)).cuda()
    ch = torch.empty(T, H, dtype=torch.float16, device="cuda")
    cl = torch.empty_like(ch)
    mx = int(np.diff(cu).max())
    B = len(cu) - 1
    st = _lib.stream_ptr()

    def plain():
        _lib.check(_lib.lib().rmu_debug_attention(hi.data_ptr(), lo.data_ptr(), cu_d.data_ptr(), B, H, heads, mx, 10,
                                                  ch.data_ptr(), cl.data_ptr(), st))

    def biased():
        _lib.check(_lib.lib().rmu_debug_attention_bias(hi.data_ptr(), lo.data_ptr(), None, None, cu_d.data_ptr(), B, H,
                                                       heads, mx, tab.data_ptr(), ch.data_ptr(), cl.data_ptr(), st))

    res = {"plain": [], "bias": []}
    for f in (plain, biased):
        for _ in range(5):
            f()
    for _ in range(5):
        for name, f in (("plain", plain), ("bias", biased)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.att_reps):
                f()
            e1.record()
            e1.synchronize()
            res[name].append(e0.elapsed_time(e1) / a.att_reps)
    p, b = statistics.median(res["plain"]), statistics.median(res["bias"])
    return {"tokens": T, "sequences": B, "plain_ms_median": p, "bias_ms_median": b, "bias_over_plain": b / p,
            "plain_ms_all": res["plain"], "bias_ms_all": res["bias"]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--bulk-reps", type=int, default=5)
    ap.add_argument("--att-reps", type=int, default=50)
    ap.add_argument("--json", default=None, help="also write the results here")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    res = {"card": card(), "models": {}}
    ms = models()
    for name, emb in ms.items():
        res["models"][name] = time_model(emb, a)
        print(json.dumps({name: res["models"][name]}), flush=True)
    from ragmeup_b200.tokenizer import synthetic_sentences
    mp = ms["mpnet all-mpnet-base-v2"]
    _, _, cu = mp._ragged(synthetic_sentences(mp.tokenizer.get_vocab(), 1000, 126, 126, seed=2))
    res["attention_768_12"] = time_attention(a, cu)
    print(json.dumps({"attention": res["attention_768_12"]}), flush=True)
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
