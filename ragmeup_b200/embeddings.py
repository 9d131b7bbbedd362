"""HuggingFaceEmbeddings drop-in (SURVEY.md §8 rows a1-a3, a5).

Same constructor and methods as ``langchain_huggingface.embeddings.HuggingFaceEmbeddings`` as the
reference uses it (``server/RAGHelper_local.py:107-117``, ``server/RAGHelper_cloud.py:90-103``):

    HuggingFaceEmbeddings(model_name=..., model_kwargs={'device': 'cuda'})
    .embed_documents(texts) -> List[List[float]]      .embed_query(text) -> List[float]

Host side mirrors langchain-huggingface 0.0.3 + sentence-transformers 2.6.1 (newline -> space,
strip, truncation=longest_first to max_seq_length; SURVEY Appendix A.1).  The reference's
length-sorted batches of 32 exist only to limit padding; batches here are ragged (no padding), so
texts are packed in input order up to a token budget — the numbers per text are the same.
The arithmetic runs in ``csrc/rmu_encoder.cu``; there is no CPU path (``device='cpu'`` raises).
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional

import numpy as np

from . import _lib
from .encoder import MAX_TOKENS_PER_CALL, BertEncoder
from .tokenizer import RaggedTokenizer, load_tokenizer, pipelined
from .weights import ModernBertConfig, MPNetConfig, Qwen3Config, XLMRConfig, resolve_model

PIPE_TEXTS = 1000     # texts per pipelined chunk of a bulk embed_documents() call


def _check_device(model_kwargs: Optional[Dict[str, Any]]) -> Optional[int]:
    dev = (model_kwargs or {}).get("device", "cuda")
    dev = str(dev)
    if dev.startswith("cuda"):
        return int(dev.split(":")[1]) if ":" in dev else None
    raise _lib.RmuError(f"device={dev!r}: ragmeup_b200 runs on CUDA (sm_90a) only; the reference's "
                        f"force_cpu/mps settings have no equivalent here")


class HuggingFaceEmbeddings:
    """H100-native stand-in for langchain_huggingface.HuggingFaceEmbeddings."""

    def __init__(self, model_name: str = "sentence-transformers/all-mpnet-base-v2",
                 cache_folder: Optional[str] = None, model_kwargs: Optional[Dict[str, Any]] = None,
                 encode_kwargs: Optional[Dict[str, Any]] = None, multi_process: bool = False,
                 show_progress: bool = False, **_: Any):
        self.model_name = model_name
        self.cache_folder = cache_folder
        self.model_kwargs = dict(model_kwargs or {})
        self.encode_kwargs = dict(encode_kwargs or {})
        self.multi_process = multi_process
        self.show_progress = show_progress
        device = _check_device(self.model_kwargs)
        cfg, w, pooling, normalize, max_len, _act, vocab_src = resolve_model(model_name, with_head=False,
                                                                               cache_folder=cache_folder)
        self.config = cfg
        self.pooling = pooling
        # sentence-transformers applies the model's own Normalize module; encode_kwargs can force it
        self.normalize = bool(normalize or self.encode_kwargs.get("normalize_embeddings", False))
        self.max_seq_length = int(max_len)
        xlmr, modern = isinstance(cfg, XLMRConfig), isinstance(cfg, ModernBertConfig)
        qwen = isinstance(cfg, Qwen3Config)
        self.tokenizer = load_tokenizer(vocab_src, cfg.vocab_size, mpnet=isinstance(cfg, MPNetConfig), xlmr=xlmr,
                                        modernbert=modern, qwen3=qwen)
        self._ragged = RaggedTokenizer(self.tokenizer, self.max_seq_length)
        # XLM-R / RoBERTa take no token types, ModernBERT and Qwen3 have none, nor has a one-row table (DistilBERT): a
        # null pointer, all zeros
        self._types = not (xlmr or modern or qwen) and cfg.type_vocab > 1
        # Qwen3: the snapshot's default prompt (config_sentence_transformers.json default_prompt_name), if it sets one
        self._prompt = cfg.prompt if qwen else ""
        self.client = BertEncoder(cfg, w, with_head=False, device=device)

    # -- tensor fast path (additional to the reference surface)
    def encode_tensor(self, texts: List[str]):
        """texts -> CUDA fp32 [n, dim] (stays on the device)."""
        torch = self.client.torch
        if len(texts) == 0:
            return torch.empty((0, self.client.embed_dim), dtype=torch.float32, device=self.client.device)
        texts = [self._prompt + t.replace("\n", " ").strip() for t in texts]
        ids, typ, cu = self._ragged(texts)
        outs = []
        for s, e in BertEncoder._chunks(cu, MAX_TOKENS_PER_CALL):
            t0, t1 = int(cu[s]), int(cu[e])
            sub_cu = (cu[s:e + 1] - cu[s]).astype(np.int32)
            outs.append(self.client.embed_tokens(ids[t0:t1], typ[t0:t1] if self._types else None, sub_cu,
                                                 int(np.max(np.diff(sub_cu))), self.pooling, self.normalize))
        return outs[0] if len(outs) == 1 else torch.cat(outs, 0)

    def _encode_host(self, texts: List[str]) -> np.ndarray:
        if len(texts) == 0:
            return np.zeros((0, self.client.embed_dim), dtype=np.float32)
        texts = [self._prompt + t.replace("\n", " ").strip() for t in texts]
        # bulk calls: WordPiece of chunk i+1 overlapped with the device encode of chunk i
        chunks = [texts[s:s + PIPE_TEXTS] for s in range(0, len(texts), PIPE_TEXTS)]
        outs = pipelined(chunks, self._ragged, lambda t: self.client.embed_host(t[0], t[1] if self._types else None, t[2],
                                                                                  self.pooling, self.normalize))
        return outs[0] if len(outs) == 1 else np.concatenate(outs, 0)

    # -- the reference surface
    def embed_documents(self, texts: List[str]) -> List[List[float]]:
        return self._encode_host(list(texts)).tolist()

    def embed_query(self, text: str) -> List[float]:
        return self.embed_documents([text])[0]

    # LangChain's async variants simply defer to the sync ones in the reference stack
    async def aembed_documents(self, texts: List[str]) -> List[List[float]]:
        return self.embed_documents(texts)

    async def aembed_query(self, text: str) -> List[float]:
        return self.embed_query(text)
