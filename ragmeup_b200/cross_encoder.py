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
Qwen3 cross-encoders take two forms.  A ``Qwen3ForSequenceClassification`` snapshot (``score.weight``) pairs as its
tokenizer makes of (query, document), truncated ``longest_first``, and its head reads the rightmost token that is not
``pad_token_id``.  A ``Qwen3ForCausalLM`` snapshot (Qwen3-Reranker) scores as its model card does, a documented
deviation from the reference (whose CrossEncoder would put an untrained ``score`` head on it): the text is
``prefix + tokens("<Instruct>: {instruction}\n<Query>: {q}\n<Document>: {d}") + suffix`` and the score P(yes) =
``exp(log_softmax([logit_no, logit_yes])[1])`` at the last token (``Qwen3RerankPrompt``).
A ColBERT checkpoint (colbert-ir/colbertv2.0, the reference README's accuracy pick) scores by late interaction instead:
``score`` returns raw MaxSim scores (``colbert.ColBERTScorer``), where the reference's CrossEncoder would put an
untrained classification head on the checkpoint (INTEGRATION.md).  ColBERT-XM (antoinelouis/colbert-xm, the README's
multilingual pick) is ColBERT on an X-MOD backbone and runs one language, chosen as ``weights.select_language`` says.
Arithmetic: ``csrc/rmu_encoder.cu``.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
from tokenizers import Tokenizer

from .embeddings import _check_device
from .encoder import BertEncoder
from .tokenizer import PairAssembler, RaggedTokenizer, load_tokenizer, pipelined
from .weights import (QWEN3_RERANK_INSTRUCTION, QWEN3_RERANK_PREFIX, QWEN3_RERANK_SUFFIX, DebertaConfig,
                      ModernBertConfig, Qwen3Config, XLMRConfig, resolve_colbert, resolve_model)

PIPE_PAIRS = 512      # pairs per pipelined chunk of a bulk score() call (one 100-pair rerank is a single chunk)


class Qwen3RerankPrompt:
    """(query, document) pairs -> Qwen3-Reranker's ragged batch: ``prefix + tokens(text) + suffix`` with ``text =
    "<Instruct>: {instruction}\n<Query>: {q}\n<Document>: {d}"`` tokenised as the snapshot's tokenizer does (its
    post-processor included) and truncated to ``max_length - len(prefix) - len(suffix)``; prefix and suffix are
    tokenised without special tokens.  Returns (ids, None, cu_seqlens)."""

    def __init__(self, tok: Tokenizer, max_length: int, instruction: str = QWEN3_RERANK_INSTRUCTION,
                 prefix: str = QWEN3_RERANK_PREFIX, suffix: str = QWEN3_RERANK_SUFFIX):
        self.instruction = instruction
        self._tok = Tokenizer.from_str(tok.to_str())
        self._tok.no_padding()
        self._tok.no_truncation()
        self.prefix = np.asarray(self._tok.encode(prefix, add_special_tokens=False).ids, dtype=np.int32)
        self.suffix = np.asarray(self._tok.encode(suffix, add_special_tokens=False).ids, dtype=np.int32)
        room = int(max_length) - len(self.prefix) - len(self.suffix)
        if room < 1:
            raise ValueError(f"Qwen3 reranker: max_length {max_length} leaves no room between its prompt's prefix and suffix")
        self._tok.enable_truncation(max_length=room, strategy="longest_first")

    def text(self, query: str, doc: str) -> str:
        return f"<Instruct>: {self.instruction}\n<Query>: {query}\n<Document>: {doc}"

    def __call__(self, queries: Sequence[str], docs: Sequence[str]):
        enc = self._tok.encode_batch([self.text(q, d) for q, d in zip(queries, docs)])
        seqs = [np.concatenate([self.prefix, np.asarray(e.ids, dtype=np.int32), self.suffix]) for e in enc]
        cu = np.zeros(len(seqs) + 1, dtype=np.int32)
        np.cumsum([len(x) for x in seqs], out=cu[1:])
        return np.concatenate(seqs).astype(np.int32), None, cu


def yes_probability(logits):
    """[n, 2] (no, yes) logits -> exp(log_softmax(.)[:, 1]), numpy float32 or a torch tensor"""
    if isinstance(logits, np.ndarray):
        x = logits.astype(np.float64)
        m = x.max(1, keepdims=True)
        lse = m[:, 0] + np.log(np.exp(x - m).sum(1))
        return np.exp(x[:, 1] - lse).astype(np.float32)
    return logits.log_softmax(1)[:, 1].exp()


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
        modern, qwen = isinstance(cfg, ModernBertConfig), isinstance(cfg, Qwen3Config)
        self.tokenizer = load_tokenizer(vocab_src, cfg.vocab_size, xlmr=xlmr, deberta=deberta, modernbert=modern,
                                        qwen3=qwen)
        self._ragged = RaggedTokenizer(self.tokenizer, self.max_length)
        if qwen and cfg.reranker:
            self._pairs = Qwen3RerankPrompt(self.tokenizer, self.max_length)
        elif qwen:
            self._pairs = lambda a, b: self._ragged(a, b)      # the tokenizer's own pair encoding, longest_first
        else:
            # pair batches assembled from cached per-text ids (identical to self._ragged(a, b); tests/test_host_logic.py)
            self._pairs = PairAssembler(self.tokenizer, self.max_length)
        # XLM-R / RoBERTa take no token types (their tokenizers return none), and DeBERTa-v3, ModernBERT, Qwen3 and a
        # one-row table (DistilBERT) have none to select: a null pointer, all zeros
        self._types = not (xlmr or deberta or modern or qwen) and cfg.type_vocab > 1
        self.client = BertEncoder(cfg, w, with_head=True, device=device)
        self._max_tokens = self.client.max_tokens_per_call

    def _post(self, logits: np.ndarray) -> np.ndarray:
        if self.activation == "yes_prob":
            return yes_probability(logits)
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
        if self.activation == "yes_prob":
            return yes_probability(logits)
        if self.activation == "sigmoid":
            logits = torch.sigmoid(logits)
        return logits[:, 0] if self.config.num_labels == 1 else logits[:, 1]
