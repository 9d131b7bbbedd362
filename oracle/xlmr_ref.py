"""Oracle: XLM-RoBERTa / RoBERTa (transformers ``XLMRobertaModel``, ``XLMRobertaForSequenceClassification``) on the CPU,
and the float64 reference of the whole encoder with their position rule.  TEST INFRASTRUCTURE ONLY (see
``oracle/__init__.py``).

What XLM-R computes that BERT does not (transformers ``models/xlm_roberta/modeling_xlm_roberta.py``):

* positions: ``padding_idx = 1``; ``create_position_ids_from_input_ids``: a token of id 1 takes position 1 and any other
  token at offset j takes 2 + j - (tokens of id 1 before it), MPNet's rule (``mpnet_ref.position_ids``);
* one token type: the tokenizers return no token types, so row 0 of the [1, H] table is added to every token;
* the classification head ``RobertaClassificationHead``: dense, tanh, out_proj on token 0, which is BERT's pooler and
  classifier under other names (``classifier.dense`` -> ``pooler.dense``, ``classifier.out_proj`` -> ``classifier``);
* no relative position bias.

``xlmr_encoder_forward`` is that forward in fp32 torch on padded batches, as ``bert_ref.bert_encoder_forward`` is
BERT's.  ``xlmr_stack_ref`` is ``mpnet_ref.mpnet_stack_ref`` with a zero bias table (the bias adds exact zeros) plus
``encoder_kernels_ref.cls_head_ref``.  Weight dicts use the canonical names of ``ragmeup_b200.weights.weight_names``.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Sequence, Tuple

import numpy as np
import torch

from . import bert_ref
from . import encoder_kernels_ref as ekr
from . import mpnet_ref

PAD_ID = 1


@dataclass
class XLMRCfg(bert_ref.BertCfg):
    vocab_size: int = 250002
    max_pos: int = 514
    type_vocab: int = 1
    ln_eps: float = 1e-5
    position_mode: int = 1
    rel_buckets: int = 0


position_ids = mpnet_ref.position_ids


def xlmr_encoder_forward(w: Dict[str, object], cfg, input_ids: torch.Tensor, attention_mask: torch.Tensor,
                         matmul=None, device=None) -> torch.Tensor:
    """[B, S] ids / mask -> last hidden state [B, S, H], fp32, padded (pad with id 1, as XLM-R's tokenizer does; the
    additive mask is finfo.min on padded keys, HF's eager path).  ``matmul(x, W)`` computes x @ W.T."""
    mm = matmul or (lambda x, W: x @ W.t())
    dev = device or "cpu"
    tw = lambda a: bert_ref._t(a, dev)  # noqa: E731
    input_ids, attention_mask = input_ids.to(dev), attention_mask.to(dev)
    B, S = input_ids.shape
    H, nh = cfg.hidden, cfg.heads
    dh = H // nh
    # HF: inputs_embeds + token_type_embeddings, then + position_embeddings
    x = (tw(w["embeddings.word_embeddings.weight"])[input_ids] + tw(w["embeddings.token_type_embeddings.weight"])[0]) + \
        tw(w["embeddings.position_embeddings.weight"])[position_ids(input_ids)]
    x = bert_ref._layer_norm(x, tw(w["embeddings.LayerNorm.weight"]), tw(w["embeddings.LayerNorm.bias"]), cfg.ln_eps)
    add_mask = (1.0 - attention_mask.to(torch.float32))[:, None, None, :] * torch.finfo(torch.float32).min
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}."
        q = mm(x, tw(w[p + "attention.self.query.weight"])) + tw(w[p + "attention.self.query.bias"])
        k = mm(x, tw(w[p + "attention.self.key.weight"])) + tw(w[p + "attention.self.key.bias"])
        v = mm(x, tw(w[p + "attention.self.value.weight"])) + tw(w[p + "attention.self.value.bias"])
        q = q.view(B, S, nh, dh).transpose(1, 2)
        k = k.view(B, S, nh, dh).transpose(1, 2)
        v = v.view(B, S, nh, dh).transpose(1, 2)
        att = torch.softmax(torch.matmul(q, k.transpose(2, 3)) * (dh ** -0.5) + add_mask, dim=-1)
        ctx = torch.matmul(att, v).transpose(1, 2).reshape(B, S, H)
        o = mm(ctx, tw(w[p + "attention.output.dense.weight"])) + tw(w[p + "attention.output.dense.bias"])
        x = bert_ref._layer_norm(o + x, tw(w[p + "attention.output.LayerNorm.weight"]),
                                 tw(w[p + "attention.output.LayerNorm.bias"]), cfg.ln_eps)
        f = bert_ref._gelu_erf(mm(x, tw(w[p + "intermediate.dense.weight"])) + tw(w[p + "intermediate.dense.bias"]))
        o = mm(f, tw(w[p + "output.dense.weight"])) + tw(w[p + "output.dense.bias"])
        x = bert_ref._layer_norm(o + x, tw(w[p + "output.LayerNorm.weight"]), tw(w[p + "output.LayerNorm.bias"]),
                                 cfg.ln_eps)
    return x


def classifier_head(w, hidden: torch.Tensor) -> torch.Tensor:
    """RobertaClassificationHead on token 0: out_proj(tanh(dense(h_0))), with the canonical names"""
    return bert_ref.classifier_head(w, hidden)


def _tok_batch(tokenizer, texts_a, texts_b, max_length: int):
    """tokenizer(..., padding=True, truncation='longest_first', max_length=...) with pad id 1 and no token types"""
    tokenizer.enable_truncation(max_length=max_length, strategy="longest_first")
    tokenizer.enable_padding(pad_id=PAD_ID, pad_token="<pad>")
    enc = tokenizer.encode_batch(list(texts_a) if texts_b is None else list(zip(texts_a, texts_b)))
    ids = torch.tensor([e.ids for e in enc], dtype=torch.long)
    mask = torch.tensor([e.attention_mask for e in enc], dtype=torch.long)
    return ids, mask


def st_encode(w, cfg, tokenizer, sentences: Sequence[str], pooling: str = "mean", normalize: bool = True,
              max_seq_length: int = 512, batch_size: int = 32, device=None) -> np.ndarray:
    """SentenceTransformer.encode with an XLM-R model (``bert_ref.st_encode``'s batching; padding with <pad> = 1)."""
    n = len(sentences)
    if n == 0:
        return np.zeros((0, cfg.hidden), dtype=np.float32)
    order = np.argsort([-len(s) for s in sentences], kind="stable")
    out = [None] * n
    with torch.no_grad():
        for s0 in range(0, n, batch_size):
            idx = order[s0:s0 + batch_size]
            ids, mask = _tok_batch(tokenizer, [sentences[i].strip() for i in idx], None, max_seq_length)
            e = bert_ref.pool(xlmr_encoder_forward(w, cfg, ids, mask, device=device), mask.to(device or "cpu"), pooling)
            if normalize:
                e = bert_ref.l2_normalize(e)
            for j, i in enumerate(idx):
                out[i] = e[j].cpu().numpy()
    return np.asarray(out, dtype=np.float32)


def hf_embed_documents(w, cfg, tokenizer, texts: Sequence[str], **kw):
    """HuggingFaceEmbeddings.embed_documents: newline -> space, encode, .tolist()"""
    return st_encode(w, cfg, tokenizer, [t.replace("\n", " ") for t in texts], **kw).tolist()


def cross_encoder_predict(w, cfg, tokenizer, pairs: Sequence[Tuple[str, str]], max_length: int = 512,
                          batch_size: int = 32, activation: str = "sigmoid", device=None) -> np.ndarray:
    """CrossEncoder.predict (sentence-transformers 2.6.1) + HuggingFaceCrossEncoder.score with an XLM-R reranker:
    input order kept, batches of 32, strip, the tokenizer's own pair tokenisation (``<s> a </s> </s> b </s>``,
    truncation longest_first to max_length, padding with 1, no token types), logits -> activation; one label -> a
    scalar per pair, else column 1."""
    if len(pairs) == 0:
        raise IndexError("cross_encoder_predict: empty input")
    outs = []
    with torch.no_grad():
        for s0 in range(0, len(pairs), batch_size):
            chunk = pairs[s0:s0 + batch_size]
            ids, mask = _tok_batch(tokenizer, [p[0].strip() for p in chunk], [p[1].strip() for p in chunk], max_length)
            logits = classifier_head(w, xlmr_encoder_forward(w, cfg, ids, mask, device=device))
            if activation == "sigmoid":
                logits = torch.sigmoid(logits)
            outs.append(logits.cpu())
    logits = torch.cat(outs, 0).numpy().astype(np.float32)
    return logits[:, 0] if cfg.num_labels == 1 else logits[:, 1]


# ------------------------------------------------------------------------------------------ float64 whole encoder

def xlmr_stack_ref(w, cfg, ids, cu, weights: str = "fp32", device=None) -> dict:
    """The whole XLM-R encoder in float64 on the ragged batch (ids [T], cu [B + 1]): ``mpnet_ref.mpnet_stack_ref``
    (position mode 1, type row 0 added to every token) with an all-zero bias table, so attention is
    ``encoder_kernels_ref.attention_ref``'s exactly, and, when w holds the head, "logits" from ``cls_head_ref``.
    weights "fp32" | "split" as there.  Returns float64 tensors on ``device``."""
    dev = torch.device(device or "cpu")
    wz = dict(w)
    wz[mpnet_ref.REL_BIAS] = torch.zeros((32, cfg.heads), dtype=torch.float64, device=dev)
    out = mpnet_ref.mpnet_stack_ref(wz, cfg, ids, cu, weights, device=dev)
    if "pooler.dense.weight" in w:
        x = out["hidden"]
        V = lambda name: ekr._f64(w[name]).to(dev)  # noqa: E731
        out["logits"] = ekr.cls_head_ref(x, torch.zeros_like(x), [int(c) for c in cu], V("pooler.dense.weight"),
                                         V("pooler.dense.bias"), V("classifier.weight"), V("classifier.bias"))[0]
    return out
