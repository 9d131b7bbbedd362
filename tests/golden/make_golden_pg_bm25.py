"""Write tests/golden/pg_bm25.npz: a seeded corpus, pg_search queries and the oracle's top-k.

    python tests/golden/make_golden_pg_bm25.py

The corpus mixes Zipf-distributed words with punctuation, hyphenated words, decimals, accents, CJK and repeated
documents; row 3 is deleted.  Scores and rows come from ``oracle/pg_bm25_ref.py`` (float32, brute force).
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import pg_bm25_ref  # noqa: E402

K = 10
QUERIES = ["w1 w5", "+w2 w7", "-w1 w3 w4", '"w1 w2"', "w1 AND w3", "w2 OR w9 OR nothing", "NOT w1 w6",
           "state-of-the-art", "café 3.5", "w0 w0 w1", "東京", "zzz", "+w1 +zzz w2"]
DELETED = (3,)


def corpus(seed: int = 0, n: int = 300):
    rng = np.random.default_rng(seed)
    words = [f"w{j}" for j in range(60)] + ["state-of-the-art", "café", "Café", "3.5", "東京", "U.S.", "naïve!"]
    p = 1.0 / (np.arange(len(words)) + 1.0)
    p /= p.sum()
    docs = [" ".join(words[j] for j in rng.choice(len(words), size=int(rng.integers(0, 40)), p=p)) for _ in range(n)]
    docs[10] = docs[11] = docs[12] = "w1 w2 w3"         # ties resolve by row
    docs[20] = ""
    return docs


def main() -> None:
    docs = corpus()
    live = [None if i in DELETED else d for i, d in enumerate(docs)]
    scores = np.zeros((len(QUERIES), K), np.float32)
    rows = np.full((len(QUERIES), K), -1, np.int64)
    for q, text in enumerate(QUERIES):
        s, r = pg_bm25_ref.search(live, pg_bm25_ref.parse(text), K)
        scores[q, :len(s)] = s
        rows[q, :len(r)] = r
    np.savez(os.path.join(os.path.dirname(os.path.abspath(__file__)), "pg_bm25.npz"),
             docs=np.frombuffer(json.dumps(docs).encode(), np.uint8),
             queries=np.frombuffer(json.dumps(QUERIES).encode(), np.uint8),
             deleted=np.asarray(DELETED, np.int64), k=np.int64(K), scores=scores, rows=rows)


if __name__ == "__main__":
    main()
