"""Time ModernBERT-base shapes on the GPU encoder, in one run:

    python tools/bench_modernbert.py [--calls 30] [--warmup 5] [--json OUT]

* the rerank call at RAGMeUp's shape, one query against 14 documents of about 128 words (gte-reranker-modernbert-base),
  and a bulk call of 64 queries x 100 such documents, both HuggingFaceCrossEncoder.score on the host clock;
* a long-document embed, 8 documents of 8192 tokens (modernbert-embed-base), host clock;
* E2 alone on that batch's QKV planes, per layer: a global layer (plain attention) and a local one (half-window 64),
  by CUDA events.
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
    ce = HuggingFaceCrossEncoder("synthetic:gte-reranker-modernbert-base")
    qs = words(a.calls + a.warmup, 10, 1)
    docs = words(14, DOC_WORDS, 2)
    t = []
    for i in range(a.calls + a.warmup):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ce.score([(qs[i], d) for d in docs])
        torch.cuda.synchronize()
        if i >= a.warmup:
            t.append(time.perf_counter() - t0)
    _ids, _typ, cu = ce._pairs([qs[0]] * 14, docs)
    bulk = [(q, d) for q in words(64, 10, 3) for d in words(100, DOC_WORDS, 4)]
    ce.score(bulk)
    bt = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ce.score(bulk)
        torch.cuda.synchronize()
        bt.append(time.perf_counter() - t0)
    res["rerank"] = {"call_1x14_ms_median": 1e3 * statistics.median(t), "call_1x14_ms_min": 1e3 * min(t),
                     "tokens_per_pair": float(np.mean(np.diff(cu))), "bulk_64x100_ms_median": 1e3 * statistics.median(bt)}
    emb = HuggingFaceEmbeddings("synthetic:modernbert-embed-base")
    cfg = emb.config
    B, S = 8, 8192
    rng = np.random.default_rng(5)
    ids = rng.integers(3, cfg.vocab_size, B * S).astype(np.int32)
    cuh = (np.arange(B + 1) * S).astype(np.int32)
    emb.client.embed_host(ids, None, cuh, "mean", True)
    et = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        emb.client.embed_host(ids, None, cuh, "mean", True)
        torch.cuda.synchronize()
        et.append(time.perf_counter() - t0)
    H, heads = cfg.hidden, cfg.heads
    x = rng.standard_normal((B * S, 3 * H)).astype(np.float32)
    x[:, :H] *= 0.2
    qkv = [torch.from_numpy(p).cuda() for p in ref.split_f16(x)]
    cu_d = torch.from_numpy(cuh).cuda()
    ch = torch.empty((B * S, H), dtype=torch.float16, device="cuda")
    cl = torch.empty_like(ch)
    lib = _lib.lib()

    def e2(window):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        args = (qkv[0].data_ptr(), qkv[1].data_ptr(), cu_d.data_ptr(), B, H, heads, S)
        run = (lambda: lib.rmu_debug_attention(*args, 10, ch.data_ptr(), cl.data_ptr(), _lib.stream_ptr())) if window == 0 \
            else (lambda: lib.rmu_debug_attention_window(*args, window, ch.data_ptr(), cl.data_ptr(), _lib.stream_ptr()))
        _lib.check(run(), "attention")
        ev[0].record()
        for _ in range(5):
            run()
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / 5

    g, l = e2(0), e2(64)
    n_local = sum(1 for w in cfg.layer_windows if w > 0)
    res["embed_8x8192"] = {"ms_median": 1e3 * statistics.median(et), "e2_global_layer_ms": g, "e2_local_layer_ms": l,
                           "global_layers": cfg.layers - n_local, "local_layers": n_local,
                           "e2_total_ms": g * (cfg.layers - n_local) + l * n_local}
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
