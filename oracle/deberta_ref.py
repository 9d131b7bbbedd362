"""Oracle: DeBERTa-v2 / v3 cross-encoders (transformers ``DebertaV2ForSequenceClassification``) on the CPU, and the
float64 reference of the whole encoder and of its disentangled attention.  TEST INFRASTRUCTURE ONLY (see
``oracle/__init__.py``).

What DeBERTa-v3 computes that BERT does not (transformers ``models/deberta_v2/modeling_deberta_v2.py``):

* embeddings: ``LN(word[id])``: no absolute positions (``position_biased_input`` false), no token types;
* one ``R = LN_rel(rel_embeddings[0:2s])`` shared by every layer (``norm_rel_ebd = layer_norm``, the encoder's
  LayerNorm);
* per layer, with ``share_att_key``: ``PQ = Wq R + bq`` and ``PK = Wk R + bk``, split by head, and
  ``score(i, j) = (Q_i.K_j + Q_i.PK[c] + K_j.PQ[c]) / sqrt(3 d)``, ``c = clamp(s + bucket(i - j), 0, 2s - 1)``
  (transformers gathers p2c at ``s - bucket(j - i)`` and transposes; bucket is odd, so it is the same c);
* ``bucket`` = ``make_log_bucket_position``, in float32;
* the head: ``classifier(gelu(pooler.dense(h_CLS)))`` (ContextPooler, erf-GELU).

``deberta_encoder_forward`` is that forward in fp32 torch on padded batches (``bert_ref.bert_encoder_forward``'s
role); ``deberta_stack_ref`` the float64 forward on the ragged batch, weights as given or as the split planes.  Weight
dicts use the canonical names of ``ragmeup_b200.weights.weight_names``.
"""
from __future__ import annotations

import math
from typing import Dict, Sequence, Tuple

import numpy as np
import torch

from . import bert_ref
from . import encoder_kernels_ref as ekr

REL_EMB = "encoder.rel_embeddings.weight"
REL_LN = ("encoder.LayerNorm.weight", "encoder.LayerNorm.bias")
PAD_ID = 0


def log_bucket(r, s: int, max_position: int) -> np.ndarray:
    """make_log_bucket_position(r, s, max_position) in its float32 arithmetic (int array in, int64 array out)"""
    r = np.asarray(r, dtype=np.int64)
    mid = s // 2
    a = np.abs(r)
    safe = np.maximum(a, 1).astype(np.float32)
    lp = np.ceil(np.log(safe / np.float32(mid)) / np.log(np.float32((max_position - 1) / mid)) * np.float32(mid - 1)) \
        + np.float32(mid)
    return np.where(a <= mid, r, np.sign(r) * lp.astype(np.int64))


def position_index(S: int, s: int, max_position: int) -> np.ndarray:
    """[S, S] c(i, j) = clamp(s + bucket(i - j), 0, 2s - 1)"""
    i = np.arange(S)
    return np.clip(s + log_bucket(i[:, None] - i[None, :], s, max_position), 0, 2 * s - 1)


def _split_heads(x: torch.Tensor, nh: int) -> torch.Tensor:
    """[..., S, H] -> [..., nh, S, d]"""
    *lead, S, H = x.shape
    return x.reshape(*lead, S, nh, H // nh).transpose(-3, -2)


def disentangled_scores(q, k, pq, pk, cidx: torch.Tensor) -> torch.Tensor:
    """q, k [nh, S, d], pq, pk [nh, 2s, d], cidx [S, S] -> unscaled q.k + q.pk[c] + k_j.pq[c]  [nh, S, S]"""
    c2p = torch.gather(q @ pk.transpose(-1, -2), -1, cidx.expand(q.shape[0], -1, -1))
    # P2C[j, c] = k_j . pq[c], read at c(i, j): row j, column c(i, j)
    p2c_full = k @ pq.transpose(-1, -2)                            # [nh, S(j), 2s]
    p2c = torch.gather(p2c_full, -1, cidx.t().expand(q.shape[0], -1, -1)).transpose(-1, -2)
    return q @ k.transpose(-1, -2) + c2p + p2c


def deberta_encoder_forward(w: Dict[str, object], cfg, input_ids: torch.Tensor, attention_mask: torch.Tensor,
                            device=None) -> torch.Tensor:
    """[B, S] ids / mask -> last hidden state [B, S, H], fp32, padded (the additive mask is finfo.min on padded keys)"""
    dev = device or "cpu"
    tw = lambda a: bert_ref._t(a, dev)  # noqa: E731
    input_ids, attention_mask = input_ids.to(dev), attention_mask.to(dev)
    B, S = input_ids.shape
    H, nh = cfg.hidden, cfg.heads
    dh = H // nh
    s = cfg.position_buckets
    x = bert_ref._layer_norm(tw(w["embeddings.word_embeddings.weight"])[input_ids], tw(w["embeddings.LayerNorm.weight"]),
                             tw(w["embeddings.LayerNorm.bias"]), cfg.ln_eps)
    x = x * attention_mask[..., None].to(x.dtype)
    R = bert_ref._layer_norm(tw(w[REL_EMB])[:2 * s], tw(w[REL_LN[0]]), tw(w[REL_LN[1]]), cfg.ln_eps)
    cidx = torch.from_numpy(position_index(S, s, cfg.max_relative_positions)).to(dev)
    add_mask = (1.0 - attention_mask.to(torch.float32))[:, None, None, :] * torch.finfo(torch.float32).min
    scale = math.sqrt(dh * 3)
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}."
        lin = lambda t, n: t @ tw(w[p + n + ".weight"]).t() + tw(w[p + n + ".bias"])  # noqa: E731
        q = _split_heads(lin(x, "attention.self.query"), nh)
        k = _split_heads(lin(x, "attention.self.key"), nh)
        v = _split_heads(lin(x, "attention.self.value"), nh)
        pq = _split_heads(lin(R, "attention.self.query"), nh)
        pk = _split_heads(lin(R, "attention.self.key"), nh)
        sc = torch.stack([disentangled_scores(q[b], k[b], pq, pk, cidx) for b in range(B)]) / scale
        att = torch.softmax(sc + add_mask, dim=-1)
        ctx = (att @ v).transpose(1, 2).reshape(B, S, H)
        o = lin(ctx, "attention.output.dense")
        x = bert_ref._layer_norm(o + x, tw(w[p + "attention.output.LayerNorm.weight"]),
                                 tw(w[p + "attention.output.LayerNorm.bias"]), cfg.ln_eps)
        f = bert_ref._gelu_erf(lin(x, "intermediate.dense"))
        o = lin(f, "output.dense")
        x = bert_ref._layer_norm(o + x, tw(w[p + "output.LayerNorm.weight"]), tw(w[p + "output.LayerNorm.bias"]),
                                 cfg.ln_eps)
    return x


def classifier_head(w, hidden: torch.Tensor) -> torch.Tensor:
    """ContextPooler + classifier on token 0: classifier(gelu(pooler.dense(h_0)))"""
    dev = hidden.device
    h0 = hidden[:, 0]
    pooled = bert_ref._gelu_erf(h0 @ bert_ref._t(w["pooler.dense.weight"], dev).t() + bert_ref._t(w["pooler.dense.bias"], dev))
    return pooled @ bert_ref._t(w["classifier.weight"], dev).t() + bert_ref._t(w["classifier.bias"], dev)


def _tok_batch(tokenizer, texts_a, texts_b, max_length: int):
    """tokenizer(a, b, padding=True, truncation='longest_first', max_length=...): pad id 0, no token types"""
    tokenizer.enable_truncation(max_length=max_length, strategy="longest_first")
    tokenizer.enable_padding(pad_id=PAD_ID, pad_token="[PAD]")
    enc = tokenizer.encode_batch(list(zip(texts_a, texts_b)))
    ids = torch.tensor([e.ids for e in enc], dtype=torch.long)
    mask = torch.tensor([e.attention_mask for e in enc], dtype=torch.long)
    return ids, mask


def cross_encoder_predict(w, cfg, tokenizer, pairs: Sequence[Tuple[str, str]], max_length: int = 512,
                          batch_size: int = 32, activation: str = "sigmoid", device=None) -> np.ndarray:
    """CrossEncoder.predict (sentence-transformers 2.6.1) + HuggingFaceCrossEncoder.score with a DeBERTa reranker:
    input order kept, batches of 32, strip, ``[CLS] a [SEP] b [SEP]``, truncation longest_first, logits ->
    activation; one label -> a scalar per pair, else column 1."""
    if len(pairs) == 0:
        raise IndexError("cross_encoder_predict: empty input")
    outs = []
    with torch.no_grad():
        for s0 in range(0, len(pairs), batch_size):
            chunk = pairs[s0:s0 + batch_size]
            ids, mask = _tok_batch(tokenizer, [p[0].strip() for p in chunk], [p[1].strip() for p in chunk], max_length)
            logits = classifier_head(w, deberta_encoder_forward(w, cfg, ids, mask, device=device))
            if activation == "sigmoid":
                logits = torch.sigmoid(logits)
            outs.append(logits.cpu())
    logits = torch.cat(outs, 0).numpy().astype(np.float32)
    return logits[:, 0] if cfg.num_labels == 1 else logits[:, 1]


# ------------------------------------------------------------------------------------------ float64 references

def disentangled_attention_ref(qkv, cu, heads: int, pos, cidx_of, cls_q=None) -> torch.Tensor:
    """float64 E2 with the position terms: qkv [T, 3H] (q pre-scaled, in log2 units), pos [2s, 2H] = PQ' | PK,
    cidx_of(S) -> [S, S] row indices of pos.  Softmax in base 2.  cls_q [B, H] (optional): query row 0 of each sequence
    from these rows -> ctx [B, H]; else ctx [T, H]."""
    qkv = qkv.double()
    pos = pos.double()
    T, H3 = qkv.shape
    H = H3 // 3
    pq, pk = _split_heads(pos[:, :H], heads), _split_heads(pos[:, H:], heads)
    cu = [int(c) for c in cu]
    B = len(cu) - 1
    out = torch.zeros((B if cls_q is not None else T, H), dtype=torch.float64, device=qkv.device)
    for b in range(B):
        t0, S = cu[b], cu[b + 1] - cu[b]
        if S == 0:
            continue
        q = _split_heads(qkv[t0:t0 + S, :H], heads)
        k = _split_heads(qkv[t0:t0 + S, H:2 * H], heads)
        v = _split_heads(qkv[t0:t0 + S, 2 * H:], heads)
        cidx = torch.as_tensor(cidx_of(S), device=qkv.device)
        if cls_q is not None:
            q = _split_heads(cls_q[b:b + 1].double(), heads).expand(-1, S, -1).clone()
        sc = disentangled_scores(q, k, pq, pk, cidx)
        p = torch.exp2(sc - sc.amax(-1, keepdim=True))
        ctx = ((p / p.sum(-1, keepdim=True)) @ v).transpose(0, 1).reshape(S, H)
        if cls_q is not None:
            out[b] = ctx[0]
        else:
            out[t0:t0 + S] = ctx
    return out


def deberta_stack_ref(w, cfg, ids, cu, weights: str = "fp32", device=None) -> dict:
    """The whole DeBERTa encoder in float64 on the ragged batch (ids [T], cu [B + 1]), weights "fp32" as given or
    "split" (hi + lo of the split planes for the GEMM weights), and the head when w holds it.  Returns {"hidden": [T, H],
    "logits": [B, num_labels]} float64 on ``device``."""
    if weights not in ("fp32", "split"):
        raise ValueError(weights)
    dev = torch.device(device or "cpu")
    Wt = lambda name: (ekr.split_weight(w[name]) if weights == "split" else ekr._f64(w[name])).to(dev)  # noqa: E731
    V = lambda name: ekr._f64(w[name]).to(dev)                                                            # noqa: E731
    cu_l = [int(c) for c in cu]
    H, heads, eps, s = cfg.hidden, cfg.heads, float(cfg.ln_eps), cfg.position_buckets
    ids_t = ekr._long(ids, dev)
    x = ekr.layernorm_ref(V("embeddings.word_embeddings.weight")[ids_t], V("embeddings.LayerNorm.weight"),
                          V("embeddings.LayerNorm.bias"), eps)[0]
    R = ekr.layernorm_ref(V(REL_EMB)[:2 * s], V(REL_LN[0]), V(REL_LN[1]), eps)[0]
    qs = math.log2(math.e) / math.sqrt(3 * (H // heads))
    cidx_of = lambda S: position_index(S, s, cfg.max_relative_positions)  # noqa: E731
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}."
        wqkv = torch.cat([Wt(p + "attention.self." + n + ".weight") for n in ("query", "key", "value")])
        bqkv = torch.cat([V(p + "attention.self." + n + ".bias") for n in ("query", "key", "value")])
        qkv = x @ wqkv.t() + bqkv
        qkv[:, :H] *= qs
        pos = R @ wqkv[:2 * H].t() + bqkv[:2 * H]
        pos[:, :H] *= qs
        ctx = disentangled_attention_ref(qkv, cu_l, heads, pos, cidx_of)
        o = ctx @ Wt(p + "attention.output.dense.weight").t() + V(p + "attention.output.dense.bias") + x
        x1 = ekr.layernorm_ref(o, V(p + "attention.output.LayerNorm.weight"), V(p + "attention.output.LayerNorm.bias"),
                               eps)[0]
        f = x1 @ Wt(p + "intermediate.dense.weight").t() + V(p + "intermediate.dense.bias")
        f = 0.5 * f * (1.0 + torch.erf(f / math.sqrt(2.0)))
        o = f @ Wt(p + "output.dense.weight").t() + V(p + "output.dense.bias") + x1
        x = ekr.layernorm_ref(o, V(p + "output.LayerNorm.weight"), V(p + "output.LayerNorm.bias"), eps)[0]
    out = {"hidden": x}
    if "pooler.dense.weight" in w:
        h0 = torch.stack([x[cu_l[b]] if cu_l[b + 1] > cu_l[b] else torch.zeros(H, dtype=torch.float64, device=dev)
                          for b in range(len(cu_l) - 1)])
        pz = h0 @ V("pooler.dense.weight").t() + V("pooler.dense.bias")
        pz = 0.5 * pz * (1.0 + torch.erf(pz / math.sqrt(2.0)))
        out["logits"] = pz @ V("classifier.weight").t() + V("classifier.bias")
    return out
