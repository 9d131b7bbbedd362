"""Oracle: post-LN BERT encoder / sequence-classification forward, pooling,
normalisation, and the sentence-transformers batching rules, restated on the
CPU in fp32 torch.  TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

What it follows (the reference itself only *calls* these; SURVEY.md §2.2):

* H3  BertModel forward — transformers ``modeling_bert.py``: embeddings sum +
  LayerNorm(eps) (``:53-113``), eager attention softmax(QK^T/sqrt(d)+mask)V
  (``:114-140``), self-attention block (``:168-208``), output / FFN blocks with
  erf-GELU and post-LayerNorm (``:287-357``).
* H9  pooler tanh(W_p h_cls + b_p) (``:456-468``) + classifier (``:1095-1125``).
* H4  sentence-transformers Pooling(mean|cls) + Normalize (Appendix A.2).
* H2  ``SentenceTransformer.encode`` (2.6.1) batching (Appendix A.1), called
  by the reference at ``server/RAGHelper_local.py:114-117`` through
  ``HuggingFaceEmbeddings.embed_documents`` (newline -> space; A.1).
* H8  ``CrossEncoder.predict`` (2.6.1) batching (Appendix A.5), called at
  ``server/RAGHelper.py:484`` through ``HuggingFaceCrossEncoder.score`` (A.6).

Weights are a plain ``dict[str, np.ndarray | torch.Tensor]`` with HuggingFace
``BertModel`` key names (no ``bert.`` prefix), plus ``pooler.dense.*`` and
``classifier.*`` for the cross-encoder.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch


@dataclass
class BertCfg:
    vocab_size: int = 30522
    hidden: int = 384
    layers: int = 6
    heads: int = 12
    ffn: int = 1536
    max_pos: int = 512
    type_vocab: int = 2
    ln_eps: float = 1e-12
    num_labels: int = 1


def _t(w, device=None) -> torch.Tensor:
    if isinstance(w, torch.Tensor):
        return w.detach().to(device=device or "cpu", dtype=torch.float32)
    return torch.from_numpy(np.ascontiguousarray(w, dtype=np.float32)).to(device or "cpu")


def _layer_norm(x: torch.Tensor, g: torch.Tensor, b: torch.Tensor, eps: float) -> torch.Tensor:
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)       # biased variance, as nn.LayerNorm
    return (x - mu) / torch.sqrt(var + eps) * g + b


def _gelu_erf(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def bert_encoder_forward(w: Dict[str, object], cfg: BertCfg, input_ids: torch.Tensor,
                         attention_mask: torch.Tensor,
                         token_type_ids: Optional[torch.Tensor] = None,
                         matmul=None, device=None) -> torch.Tensor:
    """[B,S] ids/mask/type -> last hidden state [B,S,H], fp32, padded computation
    (additive mask = finfo.min on padded keys, exactly the HF eager path).

    ``matmul(x, W)`` computes ``x @ W.T``; tests swap it to emulate reduced
    precision when sizing tolerances.  ``device`` (default the CPU) is where the
    forward runs; the result stays there."""
    mm = matmul or (lambda x, W: x @ W.t())
    dev = device or "cpu"
    tw = lambda a: _t(a, dev)  # noqa: E731
    input_ids, attention_mask = input_ids.to(dev), attention_mask.to(dev)
    B, S = input_ids.shape
    H, nh = cfg.hidden, cfg.heads
    dh = H // nh
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    token_type_ids = token_type_ids.to(dev)
    pos = torch.arange(S, device=dev)
    x = (tw(w["embeddings.word_embeddings.weight"])[input_ids]
         + tw(w["embeddings.token_type_embeddings.weight"])[token_type_ids]
         + tw(w["embeddings.position_embeddings.weight"])[pos][None])
    x = _layer_norm(x, tw(w["embeddings.LayerNorm.weight"]), tw(w["embeddings.LayerNorm.bias"]), cfg.ln_eps)
    add_mask = (1.0 - attention_mask.to(torch.float32))[:, None, None, :] * torch.finfo(torch.float32).min
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}."
        q = mm(x, tw(w[p + "attention.self.query.weight"])) + tw(w[p + "attention.self.query.bias"])
        k = mm(x, tw(w[p + "attention.self.key.weight"])) + tw(w[p + "attention.self.key.bias"])
        v = mm(x, tw(w[p + "attention.self.value.weight"])) + tw(w[p + "attention.self.value.bias"])
        q = q.view(B, S, nh, dh).transpose(1, 2)
        k = k.view(B, S, nh, dh).transpose(1, 2)
        v = v.view(B, S, nh, dh).transpose(1, 2)
        att = torch.matmul(q, k.transpose(2, 3)) * (dh ** -0.5) + add_mask
        att = torch.softmax(att, dim=-1)
        ctx = torch.matmul(att, v).transpose(1, 2).reshape(B, S, H)
        o = mm(ctx, tw(w[p + "attention.output.dense.weight"])) + tw(w[p + "attention.output.dense.bias"])
        x = _layer_norm(o + x, tw(w[p + "attention.output.LayerNorm.weight"]),
                        tw(w[p + "attention.output.LayerNorm.bias"]), cfg.ln_eps)
        f = _gelu_erf(mm(x, tw(w[p + "intermediate.dense.weight"])) + tw(w[p + "intermediate.dense.bias"]))
        o = mm(f, tw(w[p + "output.dense.weight"])) + tw(w[p + "output.dense.bias"])
        x = _layer_norm(o + x, tw(w[p + "output.LayerNorm.weight"]), tw(w[p + "output.LayerNorm.bias"]), cfg.ln_eps)
    return x


def pool(hidden: torch.Tensor, attention_mask: torch.Tensor, mode: str) -> torch.Tensor:
    """sentence-transformers Pooling (Appendix A.2)."""
    if mode == "cls":
        return hidden[:, 0]
    if mode == "mean":
        m = attention_mask[..., None].to(torch.float32)
        return (hidden * m).sum(1) / torch.clamp(m.sum(1), min=1e-9)
    raise ValueError(mode)


def l2_normalize(x: torch.Tensor) -> torch.Tensor:
    """F.normalize(x, p=2, dim=1): x / max(||x||, 1e-12)."""
    return x / torch.clamp_min(x.norm(dim=1, keepdim=True), 1e-12)


def classifier_head(w: Dict[str, object], hidden: torch.Tensor) -> torch.Tensor:
    """BertForSequenceClassification head: pooler tanh + classifier -> [B, num_labels], on hidden's device."""
    dev = hidden.device
    pooled = torch.tanh(hidden[:, 0] @ _t(w["pooler.dense.weight"], dev).t() + _t(w["pooler.dense.bias"], dev))
    return pooled @ _t(w["classifier.weight"], dev).t() + _t(w["classifier.bias"], dev)


# --------------------------------------------------------------------------- host-side batching rules

def _tok_batch(tokenizer, texts_a: Sequence[str], texts_b: Optional[Sequence[str]], max_length: int):
    """tokenizer(..., padding=True, truncation='longest_first', max_length=...) with a
    raw ``tokenizers.Tokenizer``.  Returns int64 ids / mask / type [B, S]."""
    tokenizer.enable_truncation(max_length=max_length, strategy="longest_first")
    tokenizer.enable_padding(pad_id=0, pad_token="[PAD]")
    if texts_b is None:
        enc = tokenizer.encode_batch(list(texts_a))
    else:
        enc = tokenizer.encode_batch(list(zip(texts_a, texts_b)))
    ids = torch.tensor([e.ids for e in enc], dtype=torch.long)
    mask = torch.tensor([e.attention_mask for e in enc], dtype=torch.long)
    typ = torch.tensor([e.type_ids for e in enc], dtype=torch.long)
    return ids, mask, typ


def st_encode(w, cfg: BertCfg, tokenizer, sentences: Sequence[str], pooling: str = "mean",
              normalize: bool = True, max_seq_length: int = 256, batch_size: int = 32) -> np.ndarray:
    """SentenceTransformer.encode (Appendix A.1): sort by -len(text), batches of 32,
    strip, pad to longest in batch, forward, pool, (Normalize module), un-sort."""
    n = len(sentences)
    order = np.argsort([-len(s) for s in sentences], kind="stable")
    out = [None] * n
    with torch.no_grad():
        for s0 in range(0, n, batch_size):
            idx = order[s0:s0 + batch_size]
            batch = [sentences[i].strip() for i in idx]
            ids, mask, typ = _tok_batch(tokenizer, batch, None, max_seq_length)
            h = bert_encoder_forward(w, cfg, ids, mask, typ)
            e = pool(h, mask, pooling)
            if normalize:
                e = l2_normalize(e)
            for j, i in enumerate(idx):
                out[i] = e[j].numpy()
    if n == 0:
        return np.zeros((0, cfg.hidden), dtype=np.float32)
    return np.asarray(out, dtype=np.float32)


def hf_embed_documents(w, cfg, tokenizer, texts: Sequence[str], **kw) -> List[List[float]]:
    """HuggingFaceEmbeddings.embed_documents (langchain-huggingface 0.0.3; H1):
    newline -> space, encode, .tolist()."""
    texts = [t.replace("\n", " ") for t in texts]
    return st_encode(w, cfg, tokenizer, texts, **kw).tolist()


def hf_embed_query(w, cfg, tokenizer, text: str, **kw) -> List[float]:
    return hf_embed_documents(w, cfg, tokenizer, [text], **kw)[0]


def cross_encoder_predict(w, cfg: BertCfg, tokenizer, pairs: Sequence[Tuple[str, str]],
                          max_length: int = 512, batch_size: int = 32,
                          activation: str = "identity") -> np.ndarray:
    """CrossEncoder.predict (Appendix A.5) + HuggingFaceCrossEncoder.score (A.6):
    input order kept, batches of 32, strip, pair-tokenise, logits -> activation;
    num_labels==1 -> scalar per pair; ndim>1 -> column 1."""
    if len(pairs) == 0:
        # ST 2.6.1 raises on an empty list (SURVEY §3.4); the oracle mirrors that.
        raise IndexError("cross_encoder_predict: empty input")
    outs = []
    with torch.no_grad():
        for s0 in range(0, len(pairs), batch_size):
            chunk = pairs[s0:s0 + batch_size]
            a = [p[0].strip() for p in chunk]
            b = [p[1].strip() for p in chunk]
            ids, mask, typ = _tok_batch(tokenizer, a, b, max_length)
            h = bert_encoder_forward(w, cfg, ids, mask, typ)
            logits = classifier_head(w, h)
            if activation == "sigmoid":
                logits = torch.sigmoid(logits)
            outs.append(logits)
    logits = torch.cat(outs, 0).numpy().astype(np.float32)
    if cfg.num_labels == 1:
        return logits[:, 0]
    return logits[:, 1]
