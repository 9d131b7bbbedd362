"""Time the Qwen3 0.6B shape on the GPU encoder, in one run:

    python tools/bench_qwen3.py [--calls 30] [--warmup 5] [--json OUT]

* the rerank call at RAGMeUp's shape (vector_store_k = 10): one query against 10 documents of 128 words through
  HuggingFaceCrossEncoder.score with the Qwen3-Reranker prompt, host clock;
* bulk embedding, 10 000 chunks of 512 characters through HuggingFaceEmbeddings.embed_documents, host clock;
* long-document embeds, 8 sequences of 8192 tokens, host clock;
* the causal grouped-query attention kernel alone on that batch's planes (16 query heads, 8 kv heads), CUDA events,
  with its rate in useful FLOP/s (4 d per visible (query, key) pair and head, the three split products not counted).
The card's name and power limit are read in the same run.  Synthetic weights: only the shapes are the models'.
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

DOC_WORDS = 128


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")] if out else ("?", "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def words(n, k, seed):
    syl = ["ba", "ce", "di", "fo", "gu", "ha", "je", "ki", "lo", "mu", "na", "pe", "qi", "ro", "su", "ta"]
    rng = np.random.default_rng(seed)
    return [" ".join("".join(syl[j] for j in rng.integers(0, 16, 2)) for _ in range(k)) for _ in range(n)]


def timed(fn, reps):
    import torch
    t = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return t


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results here")
    a = ap.parse_args()
    import torch
    from oracle import encoder_kernels_ref as ref
    from ragmeup_b200 import _lib
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    res = {"card": card()}

    ce = HuggingFaceCrossEncoder("synthetic:qwen3-reranker-0.6b")
    qs = words(a.calls + a.warmup, 10, 1)
    docs = words(10, DOC_WORDS, 2)
    t = []
    for i in range(a.calls + a.warmup):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ce.score([(qs[i], d) for d in docs])
        torch.cuda.synchronize()
        if i >= a.warmup:
            t.append(time.perf_counter() - t0)
    _ids, _typ, cu = ce._pairs([qs[0]] * 10, docs)
    res["rerank_1x10"] = {"ms_median": 1e3 * statistics.median(t), "ms_min": 1e3 * min(t),
                          "tokens_per_pair": float(np.mean(np.diff(cu)))}
    del ce
    torch.cuda.empty_cache()

    emb = HuggingFaceEmbeddings("synthetic:qwen3-embedding-0.6b")
    rng = np.random.default_rng(3)
    chunks = [" ".join(words(1, 200, int(s))[0].split())[:512] for s in rng.integers(0, 1 << 30, 10000)]
    emb.embed_documents(chunks[:1000])
    bt = timed(lambda: emb.embed_documents(chunks), 2)
    _i, _t, ccu = emb._ragged(chunks[:1000])
    res["embed_10000x512chars"] = {"s_median": statistics.median(bt), "chunks_per_s": 10000 / statistics.median(bt),
                                   "tokens_per_chunk": float(np.mean(np.diff(ccu)))}

    cfg = emb.config
    B, S = 8, 8192
    ids = rng.integers(3, cfg.vocab_size, B * S).astype(np.int32)
    cuh = (np.arange(B + 1) * S).astype(np.int32)
    emb.client.embed_host(ids, None, cuh, "last", True)
    et = timed(lambda: emb.client.embed_host(ids, None, cuh, "last", True), 3)
    heads, kv, d = cfg.heads, cfg.kv_heads, cfg.head_dim
    x = rng.standard_normal((B * S, (heads + 2 * kv) * d)).astype(np.float32)
    x[:, :heads * d] *= 0.3
    qkv = [torch.from_numpy(p).cuda() for p in ref.split_f16(x)]
    cu_d = torch.from_numpy(cuh).cuda()
    ch = torch.empty((B * S, heads * d), dtype=torch.float16, device="cuda")
    cl = torch.empty_like(ch)
    lib = _lib.lib()

    def att():
        return lib.rmu_debug_attention_causal(qkv[0].data_ptr(), qkv[1].data_ptr(), cu_d.data_ptr(), B, heads, kv, S,
                                              ch.data_ptr(), cl.data_ptr(), _lib.stream_ptr())
    _lib.check(att(), "attention_causal")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(10):
        att()
    ev[1].record()
    torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / 10
    flops = 4.0 * d * heads * B * S * (S + 1) / 2
    res["embed_8x8192"] = {"ms_median": 1e3 * statistics.median(et), "attention_layer_ms": ms,
                           "attention_all_layers_ms": ms * cfg.layers, "attention_useful_tflops": flops / ms / 1e9}
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
