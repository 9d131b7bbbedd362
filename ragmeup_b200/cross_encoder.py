"""HuggingFaceCrossEncoder drop-in (SURVEY.md §8 rows a9, a10).

Same surface as ``langchain_community.cross_encoders.HuggingFaceCrossEncoder`` as the reference
constructs it (``server/RAGHelper.py:483-486``): ``HuggingFaceCrossEncoder(model_name=...)`` and
``.score(text_pairs) -> float32 array [n]``.  Host side mirrors sentence-transformers 2.6.1
``CrossEncoder.predict`` (strip, pair tokenisation ``[CLS] q [SEP] d [SEP]`` with token types 0/1,
truncation=longest_first to 512, input order kept, default activation from the model config;
SURVEY Appendix A.5/A.6).  XLM-R / RoBERTa rerankers (the bge rerankers, this class's default model) pair as
``<s> q </s> </s> d </s>`` with no token types and truncate to ``min(model_max_length, max_pos - 2)``.  DeBERTa-v2 / v3
rerankers (mxbai-rerank-*-v1) pair as ``[CLS] q [SEP] d [SEP]`` and send no token types (the model has none); they
truncate to ``min(model_max_length, max_position_embeddings)`` and run in calls of at most ``deberta_tokens_per_call``
tokens, which bounds the attention position terms' workspace.  ModernBERT rerankers (gte-reranker-modernbert-base) pair
the same way, send no token types and truncate to ``min(model_max_length, max_position_embeddings)`` (8192); their head
pools by ``classifier_pooling`` (CLS or mean).
A ColBERT checkpoint (colbert-ir/colbertv2.0, the reference README's accuracy pick) scores by late interaction instead:
``score`` returns raw MaxSim scores (``colbert.ColBERTScorer``), where the reference's CrossEncoder would put an
untrained classification head on the checkpoint (INTEGRATION.md).  ColBERT-XM (antoinelouis/colbert-xm, the README's
multilingual pick) is ColBERT on an X-MOD backbone and runs one language, chosen as ``weights.select_language`` says.
Arithmetic: ``csrc/rmu_encoder.cu``.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from .embeddings import _check_device
from .encoder import BertEncoder
from .tokenizer import PairAssembler, RaggedTokenizer, load_tokenizer, pipelined
from .weights import DebertaConfig, ModernBertConfig, XLMRConfig, resolve_colbert, resolve_model

PIPE_PAIRS = 512      # pairs per pipelined chunk of a bulk score() call (one 100-pair rerank is a single chunk)


class BaseCrossEncoder:
    """Interface of langchain.retrievers.document_compressors.cross_encoder.BaseCrossEncoder."""

    def score(self, text_pairs: List[Tuple[str, str]]) -> List[float]:
        raise NotImplementedError


class HuggingFaceCrossEncoder(BaseCrossEncoder):
    def __init__(self, model_name: str = "BAAI/bge-reranker-base", model_kwargs: Optional[Dict[str, Any]] = None,
                 cache_folder: Optional[str] = None, **_: Any):
        self.model_name = model_name
        self.model_kwargs = dict(model_kwargs or {})
        device = _check_device(self.model_kwargs)
        self.colbert = None
        cb = resolve_colbert(model_name, cache_folder=cache_folder)
        if cb is not None:
            from .colbert import ColBERTScorer
            cfg, w, linear, spec, vocab_src = cb
            self.config = cfg
            tok = load_tokenizer(vocab_src, cfg.vocab_size, xlmr=isinstance(cfg, XLMRConfig))
            self.colbert = ColBERTScorer(cfg, w, linear, spec, tok, device=device)
            self.tokenizer = self.colbert.tokenizer
            self.max_length = spec.doc_maxlen
            self.activation = "identity"
            self.client = self.colbert
            return
        cfg, w, _pool, _norm, max_len, activation, vocab_src = resolve_model(model_name, with_head=True,
                                                                             cache_folder=cache_folder)
        self.config = cfg
        self.max_length = min(int(max_len), cfg.max_pos)
        self.activation = activation
        xlmr, deberta = isinstance(cfg, XLMRConfig), isinstance(cfg, DebertaConfig)
        modern = isinstance(cfg, ModernBertConfig)
        self.tokenizer = load_tokenizer(vocab_src, cfg.vocab_size, xlmr=xlmr, deberta=deberta, modernbert=modern)
        self._ragged = RaggedTokenizer(self.tokenizer, self.max_length)
        # pair batches assembled from cached per-text ids (identical to self._ragged(a, b); tests/test_host_logic.py)
        self._pairs = PairAssembler(self.tokenizer, self.max_length)
        # XLM-R / RoBERTa take no token types (their tokenizers return none), and DeBERTa-v3 and ModernBERT have no
        # token-type table: a null pointer, all zeros
        self._types = not (xlmr or deberta or modern)
        self.client = BertEncoder(cfg, w, with_head=True, device=device)
        self._max_tokens = self.client.max_tokens_per_call

    def _post(self, logits: np.ndarray) -> np.ndarray:
        if self.activation == "sigmoid":
            logits = 1.0 / (1.0 + np.exp(-logits.astype(np.float32)))
        # num_labels == 1 -> scalar per pair; otherwise langchain takes column 1
        return np.ascontiguousarray(logits[:, 0] if self.config.num_labels == 1 else logits[:, 1], dtype=np.float32)

    def score(self, text_pairs: Sequence[Tuple[str, str]]) -> np.ndarray:
        if self.colbert is not None:
            return self.colbert.score(text_pairs)
        pairs = list(text_pairs)
        if len(pairs) == 0:
            # sentence-transformers 2.6.1 raises on an empty list (SURVEY §3.4); keep the behaviour
            raise IndexError("score() received no text pairs")
        # bulk calls: pairs in chunks, WordPiece of chunk i+1 overlapped with the device scoring of chunk i
        chunks = [pairs[s:s + PIPE_PAIRS] for s in range(0, len(pairs), PIPE_PAIRS)]
        outs = pipelined(chunks, lambda c: self._pairs([p[0].strip() for p in c], [p[1].strip() for p in c]),
                         lambda t: self.client.classify_host(t[0], t[1] if self._types else None, t[2]))
        return self._post(outs[0] if len(outs) == 1 else np.concatenate(outs, 0))

    def score_tensor(self, text_pairs: Sequence[Tuple[str, str]]):
        """same scores as a CUDA fp32 tensor [n] (stays on the device)."""
        if self.colbert is not None:
            return self.colbert.score_tensor(text_pairs)
        torch = self.client.torch
        pairs = list(text_pairs)
        if len(pairs) == 0:
            raise IndexError("score_tensor() received no text pairs")
        a = [p[0].strip() for p in pairs]
        b = [p[1].strip() for p in pairs]
        ids, typ, cu = self._pairs(a, b)
        outs = []
        for s, e in BertEncoder._chunks(cu, self._max_tokens):
            t0, t1 = int(cu[s]), int(cu[e])
            sub_cu = (cu[s:e + 1] - cu[s]).astype(np.int32)
            outs.append(self.client.classify_tokens(ids[t0:t1], typ[t0:t1] if self._types else None, sub_cu,
                                                    int(np.max(np.diff(sub_cu)))))
        logits = outs[0] if len(outs) == 1 else torch.cat(outs, 0)
        if self.activation == "sigmoid":
            logits = torch.sigmoid(logits)
        return logits[:, 0] if self.config.num_labels == 1 else logits[:, 1]
