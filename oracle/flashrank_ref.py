"""Oracle for the FlashrankRerank drop-in.  TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

Restates flashrank's ``Ranker.rerank`` and langchain-community 0.2.10's ``FlashrankRerank.compress_documents``
(``server/RAGHelper.py:11,480``) **[3P-recall]**: neither package is installed here and their sources are not in the
reference, so this follows their published code as recalled.  PARITY STATUS: unpinned (no FlashRank in this image).

* ``Ranker.rerank``: one batch of ``(query, passage["text"])`` pairs, no strip, truncation ``longest_first``; float32
  logits; ``1 / (1 + np.exp(-logits.flatten()))`` for one label, ``np.exp(l)[:, 1] / np.sum(np.exp(l), axis=1)``
  otherwise; ``passage["score"] = score``; ``passages.sort(key=lambda x: x["score"], reverse=True)``.
* ``compress_documents``: passages ``{"id": i, "text": page_content, "meta": metadata}``, ``[:top_n]``, then
  ``score >= score_threshold``, then new documents with ``{prefix+"id", prefix+"relevance_score", **meta}``.

The logits are ``bert_ref``'s fp32 forward of the padded batch (``logits_ref``), or any callable that returns them.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Sequence

import numpy as np
import torch

from oracle import bert_ref


def scores(logits: np.ndarray) -> np.ndarray:
    logits = np.asarray(logits, dtype=np.float32)
    if logits.shape[1] == 1:
        return 1 / (1 + np.exp(-logits.flatten()))
    exp_logits = np.exp(logits)
    return exp_logits[:, 1] / np.sum(exp_logits, axis=1)


def rerank(query: str, passages: List[Dict[str, Any]], logits_fn: Callable[[str, List[str]], np.ndarray]):
    logits = logits_fn(query, [p["text"] for p in passages])
    for score, passage in zip(scores(logits), passages):
        passage["score"] = score
    passages.sort(key=lambda x: x["score"], reverse=True)
    return passages


def compress_documents(documents: Sequence[Any], query: str, logits_fn, top_n: int = 3, score_threshold: float = 0.0,
                       prefix_metadata: str = "", make_doc: Callable[[str, dict], Any] = lambda t, m: (t, m)):
    passages = [{"id": i, "text": doc.page_content, "meta": doc.metadata} for i, doc in enumerate(documents)]
    out = []
    for r in rerank(query, passages, logits_fn)[:top_n]:
        if r["score"] >= score_threshold:
            out.append(make_doc(r["text"], {prefix_metadata + "id": r["id"],
                                            prefix_metadata + "relevance_score": r["score"], **r["meta"]}))
    return out


def logits_ref(w, cfg: bert_ref.BertCfg, tokenizer, query: str, texts: Sequence[str], max_length: int) -> np.ndarray:
    """float32 [n, num_labels]: the fp32 forward + classifier head of the unstripped pairs, padded to the batch's
    longest (FlashRank pads; the mask keeps padded keys out)."""
    with torch.no_grad():
        ids, mask, typ = bert_ref._tok_batch(tokenizer, [query] * len(texts), list(texts), max_length)
        h = bert_ref.bert_encoder_forward(w, cfg, ids, mask, typ)
        return bert_ref.classifier_head(w, h).numpy().astype(np.float32)


class FlashrankRerank:
    """compress_documents over a logits callable, for code that takes a compressor object (rerank provenance)."""

    def __init__(self, logits_fn, top_n: int = 3, score_threshold: float = 0.0, prefix_metadata: str = "",
                 make_doc: Callable[[str, dict], Any] = lambda t, m: (t, m)):
        self.logits_fn, self.top_n, self.score_threshold = logits_fn, top_n, score_threshold
        self.prefix_metadata, self.make_doc = prefix_metadata, make_doc

    def compress_documents(self, documents, query):
        return compress_documents(documents, query, self.logits_fn, self.top_n, self.score_threshold,
                                  self.prefix_metadata, self.make_doc)
