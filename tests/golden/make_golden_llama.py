"""Writes tests/golden/llama.npz from the float64 decoder oracle (``oracle/decoder_attention_ref.py``) on the seeded
weights of the ``tiny-llama`` shape (llama3 rope scaling, no q / k norm, two query heads per kv head), for a chat-shaped
thread tokenised by a byte-level BPE built here:

* ``ids``: the thread's tokens; ``query_ids`` / ``answer_ids`` / ``doc_ids`` (+ ``doc_cu``): its parts;
* ``hidden``: the final hidden state [T, H] (float64 forward, stored as float32);
* ``spans``: the parts' token spans as the reference slices them (query, answer, documents), [start, end);
* ``mass``: the last layer's attention summed over heads and each (row span, column span) pair, float64 [n, n];
* ``scores_q`` / ``scores_noq``: the reference's document scores with and without the query blocks, float64.

    python tests/golden/make_golden_llama.py

The zip entries have fixed timestamps, so rerunning the script writes the same bytes.
"""
from __future__ import annotations

import io
import os
import sys
import zipfile
from dataclasses import asdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import decoder_attention_ref as da  # noqa: E402
from ragmeup_b200.tokenizer import build_byte_bpe  # noqa: E402
from ragmeup_b200.weights import DECODER_PRESETS, LlamaConfig, synthetic_llama_weights  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "llama.npz")
WORDS = ["system", "user", "assistant", "question", "answer", "document", "the", "capital", "of", "France", "is",
         "Paris", "river", "Seine", "flows", "through", "Berlin", "Germany", "context", "from"]
SEED, SCALE = 3, 2.0
MODEL = f"synthetic:tiny-llama:{SEED}:{SCALE}"        # the same weights through resolve_decoder


def tokenizer():
    from transformers import PreTrainedTokenizerFast
    return PreTrainedTokenizerFast(tokenizer_object=build_byte_bpe(WORDS))


def thread():
    """(thread, query, documents, answer): a system prompt holding the documents, then the user turn and the answer"""
    docs = [f"document {i}: the river Seine flows through Paris " + "the capital " * (3 * i) + f"{i}" for i in range(4)]
    docs.append("Berlin")                                   # a one-token part: an empty slice, a NaN score
    query = "question: what is the capital of France"
    answer = "answer: the capital of France is Paris"
    text = ("<|im_start|>system\nanswer the question from the context\n" + "\n".join(docs) + "<|im_end|>\n"
            f"<|im_start|>user\n{query}<|im_end|>\n<|im_start|>assistant\n{answer}<|im_end|>\n")
    return text, query, docs, answer


def build():
    cfg = LlamaConfig(**asdict(DECODER_PRESETS["tiny-llama"]))
    return cfg, synthetic_llama_weights(cfg, seed=SEED, scale=SCALE)


def span(ids, part):
    """the reference's slice of a part, [start : start + len - 1], as Python normalises it -> [start, end)"""
    s, e = da.find_part(ids, part)
    s, e, _ = slice(s, e).indices(len(ids))
    return s, max(s, e)


def compute():
    cfg, w = build()
    tok = tokenizer()
    text, query, docs, answer = thread()
    enc = lambda t: tok.encode(t, add_special_tokens=False)       # noqa: E731
    ids, q, a, ds = enc(text), enc(query), enc(answer), [enc(d) for d in docs]
    W = {k: torch.from_numpy(v).double() for k, v in w.items()}
    with torch.no_grad():
        hidden = da.hidden(W, cfg, ids, qk_norm=False).numpy()
        A = da.last_attention(W, cfg, ids, qk_norm=False).numpy()
    spans = [span(ids, q), span(ids, a)] + [span(ids, d) for d in ds]
    mass = np.array([[A[:, r0:r1, c0:c1].sum() for c0, c1 in spans] for r0, r1 in spans], dtype=np.float64)
    doc_cu = np.zeros(len(ds) + 1, np.int32)
    np.cumsum([len(d) for d in ds], out=doc_cu[1:])
    return {"ids": np.asarray(ids, np.int32), "query_ids": np.asarray(q, np.int32), "answer_ids": np.asarray(a, np.int32),
            "doc_ids": np.concatenate([np.asarray(d, np.int32) for d in ds]), "doc_cu": doc_cu,
            "hidden": hidden.astype(np.float32), "spans": np.asarray(spans, np.int32), "mass": mass,
            "scores_q": np.asarray(da.attention_scores(A, ids, q, a, ds, include_query=True), np.float64),
            "scores_noq": np.asarray(da.attention_scores(A, ids, q, a, ds, include_query=False), np.float64)}


def write(arrays, path=OUT):
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            b = io.BytesIO()
            np.save(b, arrays[k], allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", date_time=(2020, 1, 1, 0, 0, 0)), b.getvalue())
    with open(path, "wb") as f:
        f.write(buf.getvalue())


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    write(compute())
    print(OUT)
