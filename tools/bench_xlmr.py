"""Time the XLM-R models on the encoder: the bge-reranker-base cross-encoder (HuggingFaceCrossEncoder's default model),
multilingual-e5-base ingest, and E2 attention at bge-m3's shape for long sequences.

    python tools/bench_xlmr.py [--calls 50] [--warmup 5] [--bulk-reps 3] [--att-reps 20] [--json OUT]

* rerank call: ``score`` on one query of about 16 tokens against 14 documents of about 130 tokens (RAGMeUp's rerank
  shape, as tools/bench_flashrank.py), --calls calls timed one by one on the host clock, each ending in a device
  synchronise.  Median and minimum.
* rerank bulk: 64 queries x 100 documents, 64 ``score`` calls of 100 pairs back to back, --bulk-reps times; pairs/s.
* tokenisation: the host SentencePiece Unigram tokenisation of the bulk's pairs through a new ``PairAssembler`` (per-text
  cache empty at its first query) and through ``RaggedTokenizer``, next to BERT WordPiece pairs of about the same token
  counts; and of the ingest's chunks.
* ingest: ``embed_documents`` on 1 000 chunks of about 130 tokens with ``synthetic:multilingual-e5-base``, --bulk-reps
  times; documents/s.
* attention: ``rmu_debug_attention`` (10 warps, the encoder's configuration) at bge-m3's shape (H 1024, 16 heads, d_h
  64) on 65 536 tokens in sequences of S = 512, 2048 and 8192; CUDA events around --att-reps launches, five rounds, the
  median reported as ns per token (one layer's attention, all heads).

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


# words per query / document: synthetic words average about 1.45 Unigram pieces, so about 16 and 130 tokens
Q_WORDS, D_WORDS = 10, 88


def texts(tok, n, words_per_text, seed):
    """seeded texts of whole words of the synthetic Unigram vocabulary"""
    words = sorted(p[1:] for p in tok.get_vocab() if p.startswith("▁") and len(p) > 2)
    rng = np.random.default_rng(seed)
    return [" ".join(words[int(j)] for j in rng.integers(0, len(words), words_per_text)) for _ in range(n)]


def _timed(f):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    f()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def rerank(a) -> dict:
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.tokenizer import PairAssembler, RaggedTokenizer, load_tokenizer, synthetic_sentences, synthetic_vocab
    ce = HuggingFaceCrossEncoder(model_name="synthetic:bge-reranker-base:0:4.0")
    queries = texts(ce.tokenizer, a.calls + a.warmup, Q_WORDS, seed=1)
    docs = texts(ce.tokenizer, 14, D_WORDS, seed=2)
    cu = ce._pairs([queries[0]] * 14, docs)[2]
    for q in queries[:a.warmup]:
        ce.score([(q, d) for d in docs])
    ts = [_timed(lambda: ce.score([(q, d) for d in docs])) for q in queries[a.warmup:]]
    bq, bd = texts(ce.tokenizer, 64, Q_WORDS, seed=3), texts(ce.tokenizer, 100, D_WORDS, seed=4)
    ce.score([(bq[0], d) for d in bd])
    bulk = [_timed(lambda: [ce.score([(q, d) for d in bd]) for q in bq]) for _ in range(a.bulk_reps)]
    # host tokenisation alone: the bulk's 6 400 pairs through a new PairAssembler (its per-text cache empty at the
    # first query, as in a server's first call on these documents), and RaggedTokenizer's pair path
    tok_pa = []
    for _ in range(a.bulk_reps):
        pa = PairAssembler(ce.tokenizer, 512)
        tok_pa.append(_timed(lambda: [pa([q] * 100, bd) for q in bq]))
    rt = RaggedTokenizer(ce.tokenizer, 512)
    tok_rt = [_timed(lambda: [rt([q] * 100, bd) for q in bq]) for _ in range(a.bulk_reps)]
    # BERT WordPiece on texts of about the same token counts (synthetic BERT words are one WordPiece token each)
    wp = load_tokenizer(None, 30522)
    vocab = synthetic_vocab(30522)
    wq, wd = synthetic_sentences(vocab, 64, 15, 15, seed=3), synthetic_sentences(vocab, 100, 128, 128, seed=4)
    wrt = RaggedTokenizer(wp, 512)
    tok_wp = [_timed(lambda: [wrt([q] * 100, wd) for q in wq]) for _ in range(a.bulk_reps)]
    tok = np.diff(cu)
    wtok = np.diff(wrt([wq[0]] * 100, wd)[2])
    return {"pair_tokens_mean": float(tok.mean()), "wordpiece_pair_tokens_mean": float(wtok.mean()),
            "call_ms_median": 1e3 * statistics.median(ts), "call_ms_min": 1e3 * min(ts), "calls": len(ts),
            "bulk_64x100_ms_median": 1e3 * statistics.median(bulk), "bulk_pairs_per_s": 6400 / statistics.median(bulk),
            "unigram_pair_assembler_first_use_ms_64x100": 1e3 * statistics.median(tok_pa),
            "unigram_ragged_pairs_ms_64x100": 1e3 * statistics.median(tok_rt),
            "wordpiece_ragged_pairs_ms_64x100": 1e3 * statistics.median(tok_wp)}


def ingest(a) -> dict:
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    emb = HuggingFaceEmbeddings(model_name="synthetic:multilingual-e5-base")
    docs = texts(emb.tokenizer, 1000, D_WORDS, seed=5)
    d_tok = float(np.mean(np.diff(emb._ragged(docs)[2])))
    emb.embed_documents(docs)
    bulk = [_timed(lambda: emb.embed_documents(docs)) for _ in range(a.bulk_reps)]
    tok = [_timed(lambda: emb._ragged(docs)) for _ in range(a.bulk_reps)]
    return {"chunk_tokens_mean": d_tok, "ingest_1000_ms_median": 1e3 * statistics.median(bulk),
            "ingest_docs_per_s": 1000 / statistics.median(bulk), "unigram_1000_chunks_ms": 1e3 * statistics.median(tok)}


def attention(a) -> dict:
    import torch
    from ragmeup_b200 import _lib
    H, heads, T = 1024, 16, 65536
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(T, 3 * H, device="cuda", generator=g)
    qkv[:, :H] *= 1.4426950408889634 / 8.0
    hi = qkv.half()
    lo = (qkv - hi.float()).half()
    ch = torch.empty(T, H, dtype=torch.float16, device="cuda")
    cl = torch.empty_like(ch)
    st = _lib.stream_ptr()
    out = {}
    for S in (512, 2048, 8192):
        B = T // S
        cu = torch.arange(0, T + 1, S, dtype=torch.int32, device="cuda")

        def run():
            _lib.check(_lib.lib().rmu_debug_attention(hi.data_ptr(), lo.data_ptr(), cu.data_ptr(), B, H, heads, S, 10,
                                                      ch.data_ptr(), cl.data_ptr(), st))
        for _ in range(3):
            run()
        ms = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.att_reps):
                run()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1) / a.att_reps)
        m = statistics.median(ms)
        out[f"S={S}"] = {"sequences": B, "ms_per_launch_median": m, "ns_per_token": 1e6 * m / T, "ms_all": ms}
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--bulk-reps", type=int, default=3)
    ap.add_argument("--att-reps", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the results here")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    res = {"card": card()}
    for name, f in (("bge-reranker-base", rerank), ("multilingual-e5-base ingest", ingest),
                    ("attention bge-m3 shape", attention)):
        res[name] = f(a)
        print(json.dumps({name: res[name]}), flush=True)
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
