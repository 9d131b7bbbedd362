"""Query latency and one-document-per-call load time of the GPU pg_search BM25 leg (PostgresBM25Retriever).

    python tools/bench_pg_bm25.py [--docs 1000000] [--load 100000] [--k 10] [--out results/bench_pg_bm25.json]

* query: 1M synthetic documents of 100-130 Zipf-distributed words (vocabulary 50 000), queries of 8-16 terms, with
  and without two 2-word phrases, k = 10 (``vector_store_k`` in the reference's ``server/.env.template``); one query
  per call, as the EnsembleRetriever issues them, and 32 per call through ``batch``.  The index is built from the
  token arrays directly (the tokenizer is not what this measures).
* load: 100 000 documents through ``add_documents([d], ids=[...])`` one at a time, as server/RAGHelper.py:459-461
  loads them, then the first search, which moves them to the device.

Prints the card name and power limit beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ragmeup_b200 import pg_search  # noqa: E402
from ragmeup_b200.documents import Document  # noqa: E402
from ragmeup_b200.pg_bm25 import PgBM25Index, PostgresBM25Retriever  # noqa: E402

VOCAB = 50_000


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        pl = f"unknown ({e})"
    return name, pl


def zipf_p():
    p = 1.0 / (np.arange(VOCAB) + 1.0)
    return p / p.sum()


def synthetic_index(n_docs, rng):
    ix = PgBM25Index()
    lens = rng.integers(100, 131, size=n_docs)
    tok = rng.choice(VOCAB, size=int(lens.sum()), p=zipf_p()).astype(np.int64)
    row = np.repeat(np.arange(n_docs, dtype=np.int64), lens)
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    pos = (np.arange(len(tok)) - np.repeat(starts, lens)).astype(np.int32)
    ix.vocab = {f"w{j}": j for j in range(VOCAB)}
    pairs = np.unique(tok * n_docs + row)
    ix._df = np.bincount(pairs // n_docs, minlength=VOCAB).astype(np.int64)
    ix._lens = lens.tolist()
    ix.n_live, ix.total_live = n_docs, int(lens.sum())
    seg = ix._segment(0, n_docs, VOCAB, tok, row, pos, pg_search.fieldnorm_id(lens))
    with ix.torch.cuda.device(ix.device):
        ix._push(seg)
    ix._alive_dirty = True
    return ix


def queries(rng, n, phrases):
    out = []
    for _ in range(n):
        m = int(rng.integers(8, 17))
        words = [f"w{j}" for j in rng.choice(VOCAB, size=m, p=zipf_p())]
        if phrases:
            words[0] = f'"{words[0]} {words[1]}"'
            words[1] = f'"{words[2]} {words[3]}"'
            del words[2:4]
        out.append(" ".join(words))
    return out


def time_calls(fn, items, warm=5):
    for x in items[:warm]:
        fn(x)
    t = []
    for x in items:
        t0 = time.perf_counter()
        fn(x)
        t.append(time.perf_counter() - t0)
    return float(np.median(t) * 1e3), float(np.percentile(t, 90) * 1e3)


def log(msg):
    print(msg, file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000, help="0 skips the query measurement")
    ap.add_argument("--load", type=int, default=100_000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    name, pl = card()
    res = {"card": name, "power_limit": pl, "docs": a.docs, "k": a.k}
    if a.docs > 0:
        t0 = time.perf_counter()
        ix = synthetic_index(a.docs, rng)
        ix.flush()
        res["index_build_s"] = time.perf_counter() - t0
        log(f"index of {a.docs} documents built in {res['index_build_s']:.1f} s")
        for phrases in (False, True):
            qs = queries(rng, 200, phrases)
            parsed = [pg_search.parse_query(q) for q in qs]
            med, p90 = time_calls(lambda c: ix.search([c], a.k), parsed)
            bt = [parsed[i:i + 32] for i in range(0, len(parsed), 32)]
            bmed, _ = time_calls(lambda b: ix.search(b, a.k), bt, warm=2)
            key = "phrases" if phrases else "terms"
            res[f"query_ms_median_{key}"], res[f"query_ms_p90_{key}"] = med, p90
            res[f"batch32_ms_median_{key}"] = bmed
            log(f"{key}: {med:.3f} ms median per query, {bmed:.3f} ms per batch of 32")
        del ix
    os.environ.pop("RMU_STORE_DIR", None)
    words = np.asarray([f"w{j}" for j in range(VOCAB)])
    lens = rng.integers(100, 131, size=a.load)
    tok = rng.choice(VOCAB, size=int(lens.sum()), p=zipf_p())
    offs = np.concatenate([[0], np.cumsum(lens)])
    docs = [Document(page_content=" ".join(words[tok[offs[i]:offs[i + 1]]]), metadata={"id": f"{i:032x}"})
            for i in range(a.load)]
    ret = PostgresBM25Retriever(connection_uri="", table_name="sparse_vectors", k=a.k)
    log("load: documents generated")
    t0 = time.perf_counter()
    for i, d in enumerate(docs):
        ret.add_documents([d], ids=[d.metadata["id"]])
        if i % 20000 == 0:
            log(f"load: {i} documents")
    res["load_one_per_call_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    ret.invoke("w1 w2 w3")
    res["first_search_after_load_s"] = time.perf_counter() - t0
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
