"""Oracle: ModernBERT encoders, rerankers and embedders (transformers ``ModernBertModel`` /
``ModernBertForSequenceClassification``) on the CPU or GPU in fp32, and the float64 reference of the whole encoder and
of its sliding-window attention.  TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

What ModernBERT computes (transformers ``models/modernbert/modeling_modernbert.py``), with x the residual stream:

* ``x = LN_emb(tok_embeddings[id])``; per layer ``x += Wo attn(LN_a(x)) + bo`` (``LN_a`` the identity in layer 0) and
  ``x += Wo2 (gelu(in) * gate) + bo2`` with ``in | gate = Wi LN_m(x) + bi``; the hidden state is ``final_norm(x)``;
* q and k rotated per head with the cos / sin of the token's position, from the float32 tables of
  ``ragmeup_b200.weights.rope_tables`` (global theta on global layers, local theta on local ones); the float64 forward
  looks its cos / sin up in the same float32 tables, only the arithmetic after the lookup is float64;
* on local layers key j is visible to query i iff ``|i - j| <= window``;
* the head: ``classifier(LN(gelu(dense(p))))``, p the CLS row or the mean of the hidden state.

Every function runs one sequence at a time (no padding).  Weight dicts use the canonical names of
``ragmeup_b200.weights.modernbert_weight_names``.
"""
from __future__ import annotations

import math
from typing import Dict

import numpy as np
import torch

from . import encoder_kernels_ref as ekr

GEMM = ("attn.Wqkv.weight", "attn.Wo.weight", "mlp.Wi.weight", "mlp.Wo.weight")


def _ln(x, g, b, eps):
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    return (x - mean) / torch.sqrt(var + eps) * g + b


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def rotate(x, cos, sin):
    """x [..., S, d] rotated with cos / sin [S, d / 2] (transformers' ``x * cos + rotate_half(x) * sin``)"""
    c = torch.cat([cos, cos], -1)
    s = torch.cat([sin, sin], -1)
    h = x.shape[-1] // 2
    rot = torch.cat([-x[..., h:], x[..., :h]], -1)
    return x * c + rot * s


def window_attention_ref(qkv, cu, heads: int, window: int) -> torch.Tensor:
    """float64 E2 with a sliding window: qkv [T, 3H] (q pre-scaled, in log2 units), key j visible to query i iff
    |i - j| <= window (0 = every key).  Softmax in base 2 -> ctx [T, H]."""
    qkv = qkv.double()
    T, H3 = qkv.shape
    H = H3 // 3
    d = H // heads
    out = torch.zeros((T, H), dtype=torch.float64, device=qkv.device)
    cu = [int(c) for c in cu]
    for b in range(len(cu) - 1):
        t0, S = cu[b], cu[b + 1] - cu[b]
        if S == 0:
            continue
        sp = lambda x: x.reshape(S, heads, d).transpose(0, 1)  # noqa: E731
        q, k, v = sp(qkv[t0:t0 + S, :H]), sp(qkv[t0:t0 + S, H:2 * H]), sp(qkv[t0:t0 + S, 2 * H:])
        sc = q @ k.transpose(-1, -2)
        if window > 0:
            i = torch.arange(S, device=qkv.device)
            sc = sc.masked_fill((i[:, None] - i[None, :]).abs() > window, float("-inf"))
        p = torch.exp2(sc - sc.amax(-1, keepdim=True))
        out[t0:t0 + S] = ((p / p.sum(-1, keepdim=True)) @ v).transpose(0, 1).reshape(S, H)
    return out


def modernbert_stack(w: Dict[str, object], cfg, ids, cu, dtype=torch.float64, weights: str = "fp32", device=None,
                     pooling: str | None = None) -> dict:
    """The whole ModernBERT encoder on the ragged batch (ids [T], cu [B + 1]) in ``dtype``, weights "fp32" as given
    or "split" (hi + lo of the split planes for the four GEMM weights), and the head when w holds it, pooled by
    ``pooling`` (default cfg.classifier_pooling).  Returns {"hidden": [T, H], "logits": [B, num_labels]} on ``device``.
    An empty sequence has no hidden rows and pools to a zero vector, as the encoder's pool_kernel does."""
    from ragmeup_b200.weights import rope_tables
    if weights not in ("fp32", "split"):
        raise ValueError(weights)
    dev = torch.device(device or "cpu")

    def W(name):
        a = w[name]
        a = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.asarray(a))
        if weights == "split" and name.endswith(GEMM):
            a = ekr.split_weight(a)
        return a.to(device=dev, dtype=dtype)

    tabs = [torch.from_numpy(t).to(device=dev, dtype=dtype) for t in rope_tables(cfg)]
    H, nh, eps = cfg.hidden, cfg.heads, float(cfg.ln_eps)
    d = H // nh
    F = cfg.ffn
    cu_l = [int(c) for c in cu]
    ids_t = torch.as_tensor(np.asarray(ids, dtype=np.int64), device=dev)
    E = W("embeddings.tok_embeddings.weight")
    hidden = torch.zeros((len(ids_t), H), dtype=dtype, device=dev)
    pooled = []
    for b in range(len(cu_l) - 1):
        t0, S = cu_l[b], cu_l[b + 1] - cu_l[b]
        if S == 0:
            pooled.append(torch.zeros(H, dtype=dtype, device=dev))
            continue
        x = _ln(E[ids_t[t0:t0 + S]], W("embeddings.norm.weight"), W("embeddings.norm.bias"), eps)
        pos = torch.arange(S, device=dev)
        i = pos
        for l in range(cfg.layers):
            p = f"layers.{l}."
            win = cfg.layer_windows[l]
            a = x if l == 0 else _ln(x, W(p + "attn_norm.weight"), W(p + "attn_norm.bias"), eps)
            qkv = a @ W(p + "attn.Wqkv.weight").t() + W(p + "attn.Wqkv.bias")
            sp = lambda t: t.reshape(S, nh, d).transpose(0, 1)  # noqa: E731
            q, k, v = sp(qkv[:, :H]), sp(qkv[:, H:2 * H]), sp(qkv[:, 2 * H:])
            cos, sin = (tabs[2], tabs[3]) if win > 0 else (tabs[0], tabs[1])
            q, k = rotate(q, cos[pos], sin[pos]), rotate(k, cos[pos], sin[pos])
            sc = (q @ k.transpose(-1, -2)) * (d ** -0.5)
            if win > 0:
                sc = sc.masked_fill((i[:, None] - i[None, :]).abs() > win, float("-inf"))
            ctx = (torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(S, H)
            x = x + ctx @ W(p + "attn.Wo.weight").t() + W(p + "attn.Wo.bias")
            m = _ln(x, W(p + "mlp_norm.weight"), W(p + "mlp_norm.bias"), eps)
            hmid = m @ W(p + "mlp.Wi.weight").t() + W(p + "mlp.Wi.bias")
            x = x + (_gelu(hmid[:, :F]) * hmid[:, F:]) @ W(p + "mlp.Wo.weight").t() + W(p + "mlp.Wo.bias")
        h = _ln(x, W("final_norm.weight"), W("final_norm.bias"), eps)
        hidden[t0:t0 + S] = h
        pooled.append(h[0] if (pooling or cfg.classifier_pooling) == "cls" else h.mean(0))
    out = {"hidden": hidden}
    if "classifier.weight" in w and pooled:
        pz = torch.stack(pooled)
        y = _gelu(pz @ W("head.dense.weight").t() + W("head.dense.bias"))
        y = _ln(y, W("head.norm.weight"), W("head.norm.bias"), eps)
        out["logits"] = y @ W("classifier.weight").t() + W("classifier.bias")
    return out
