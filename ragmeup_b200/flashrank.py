"""FlashrankRerank drop-in: the reference's default reranker (``rerank_model=flashrank``, ``server/.env.template:43``).

``server/RAGHelper.py:476-480`` builds ``FlashrankRerank(top_n=self.rerank_k)`` from
``langchain.retrievers.document_compressors`` and uses it for ``rerank_retriever`` (``:488-490``) and for rerank
provenance (``server/RAGHelper_local.py:300-308`` -> ``server/provenance.py:100-108``).

The surface and host rules restate langchain-community 0.2.10's ``FlashrankRerank`` over flashrank's
``Ranker.rerank`` **[3P-recall]**: neither package is installed here and their sources are not in the reference, so
what follows is recalled from their published code, as SURVEY Appendix A does for the other wheels.

* passages ``{"id": i, "text": doc.page_content, "meta": doc.metadata}``; pairs ``(query, text)`` with no ``strip()``,
  truncation ``longest_first`` to ``min(tokenizer_config model_max_length, 512)``;
* scores in numpy float32 on the float32 logits: ``1 / (1 + exp(-l))`` for one label, ``exp(l)[:, 1] / sum(exp(l))``
  for more (no max subtraction: an overflowing exponential gives NaN, as in FlashRank).  The model config's
  ``sbert_ce_default_activation_function`` is ignored;
* ``list.sort(key=score, reverse=True)``, then ``[:top_n]``, then scores ``< score_threshold`` are dropped;
* each result is a new Document with ``metadata = {prefix+"id": i, prefix+"relevance_score": score, **meta}``.

The logits come from the sm_90a encoder (``rmu_encoder_classify_host``); the score transform is FlashRank's own
numpy arithmetic on at most ``n`` floats, so equal logits give bit-equal scores.  FlashRank runs int8-quantised ONNX
files for some models; this runs the fp32 checkpoint they were exported from (INTEGRATION.md).
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence

import numpy as np

from .documents import Document
from .encoder import BertEncoder
from .tokenizer import PairAssembler, load_tokenizer, pipelined
from .weights import resolve_flashrank

DEFAULT_MODEL_NAME = "ms-marco-MultiBERT-L-12"      # langchain-community's default [3P-recall]
PIPE_PAIRS = 512                                     # pairs per pipelined chunk of a bulk rerank


def flashrank_scores(logits: np.ndarray) -> np.ndarray:
    """FlashRank's activation on float32 logits [n, num_labels] -> float32 [n] [3P-recall: Ranker.rerank]."""
    logits = np.asarray(logits, dtype=np.float32)
    if logits.shape[1] == 1:
        return 1 / (1 + np.exp(-logits.flatten()))
    exp_logits = np.exp(logits)
    return exp_logits[:, 1] / np.sum(exp_logits, axis=1)


class RerankRequest:
    """flashrank.RerankRequest: a query and a list of passage dicts (``"id"``, ``"text"``, ``"meta"``)."""

    def __init__(self, query: Optional[str] = None, passages: Optional[List[Dict[str, Any]]] = None):
        self.query = query
        self.passages = passages if passages is not None else []


class Ranker:
    """GPU stand-in for ``flashrank.Ranker``: one model on the device, shared by any number of threads (the encoder
    handle serialises device work under its mutex; the pair cache has its own lock).  ``cache_dir`` is where the
    snapshot is looked up (``weights.resolve_flashrank``); nothing is downloaded."""

    def __init__(self, model_name: str = DEFAULT_MODEL_NAME, cache_dir: Optional[str] = None, max_length: int = 512,
                 **_: Any):
        self.model_name = model_name
        cfg, w, max_len, vocab_src = resolve_flashrank(model_name, cache_folder=cache_dir, max_length=max_length)
        self.config = cfg
        self.max_length = int(max_len)
        self.tokenizer = load_tokenizer(vocab_src, cfg.vocab_size)
        self._pairs = PairAssembler(self.tokenizer, self.max_length)
        self.encoder = BertEncoder(cfg, w, with_head=True)

    def logits(self, query: str, texts: Sequence[str]) -> np.ndarray:
        """float32 [n, num_labels] logits of the pairs (query, text), texts taken as they are (no strip)."""
        texts = list(texts)
        chunks = [texts[s:s + PIPE_PAIRS] for s in range(0, len(texts), PIPE_PAIRS)]
        outs = pipelined(chunks, lambda c: self._pairs([query] * len(c), c), lambda t: self.encoder.classify_host(*t))
        return outs[0] if len(outs) == 1 else np.concatenate(outs, 0)

    def rerank(self, request: RerankRequest) -> List[Dict[str, Any]]:
        passages = request.passages
        if len(passages) == 0:
            # FlashRank's ONNX session rejects an empty batch; ContextualCompressionRetriever never passes one
            raise ValueError("rerank() received no passages")
        scores = flashrank_scores(self.logits(request.query, [p["text"] for p in passages]))
        for score, passage in zip(scores, passages):
            passage["score"] = score
        passages.sort(key=lambda x: x["score"], reverse=True)
        return passages


def compress(client: Any, documents: Sequence[Any], query: str, top_n: int, score_threshold: float,
             prefix_metadata: str) -> List[Any]:
    """``FlashrankRerank.compress_documents`` [3P-recall]: the plain and the pydantic class both run this."""
    passages = [{"id": i, "text": doc.page_content, "meta": doc.metadata} for i, doc in enumerate(documents)]
    rerank_response = client.rerank(RerankRequest(query=query, passages=passages))[:top_n]
    final_results = []
    for r in rerank_response:
        if r["score"] >= score_threshold:
            final_results.append(Document(page_content=r["text"],
                                          metadata={prefix_metadata + "id": r["id"],
                                                    prefix_metadata + "relevance_score": r["score"], **r["meta"]}))
    return final_results


class FlashrankRerank:
    """Document compressor with the fields of langchain-community's FlashrankRerank: ``client`` (a ``Ranker``, built
    from ``model`` when not given), ``top_n``, ``score_threshold``, ``model`` (None: ``DEFAULT_MODEL_NAME``) and
    ``prefix_metadata``.  Other keyword arguments raise, as its pydantic ``extra="forbid"`` does."""

    def __init__(self, client: Any = None, top_n: int = 3, score_threshold: float = 0.0, model: Optional[str] = None,
                 prefix_metadata: str = "", **extra: Any):
        if extra:
            raise TypeError(f"unexpected fields: {sorted(extra)}")
        self.model = model
        self.client = client if client is not None else Ranker(model_name=model or DEFAULT_MODEL_NAME)
        self.top_n = int(top_n)
        self.score_threshold = float(score_threshold)
        self.prefix_metadata = str(prefix_metadata)

    def compress_documents(self, documents: Sequence[Any], query: str, callbacks: Optional[Any] = None) -> List[Any]:
        return compress(self.client, documents, query, self.top_n, self.score_threshold, self.prefix_metadata)

    async def acompress_documents(self, documents: Sequence[Any], query: str, callbacks: Optional[Any] = None) -> List[Any]:
        return self.compress_documents(documents, query, callbacks)
