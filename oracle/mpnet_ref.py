"""Oracle: MPNet (transformers ``MPNetModel``) on the CPU, and float64 references of the two encoder kernels MPNet
adds to BERT's.  TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

What MPNet computes that BERT does not (transformers ``models/mpnet/modeling_mpnet.py``):

* positions: ``padding_idx = 1`` is fixed; ``position_ids = cumsum(ids != 1) * (ids != 1) + 1``, so a token of id 1 takes
  position 1 and any other token at offset j takes 2 + j - (tokens of id 1 before it);
* no token-type embeddings: ``LayerNorm(word + position)``;
* a relative position bias ``encoder.relative_attention_bias.weight`` [32, heads], shared by all layers, added to the
  scaled scores before the mask: ``bias[bucket(j - i), h]`` with i, j from ``arange`` (not from the positions) and
  ``relative_position_bucket(num_buckets=32, max_distance=128)``.

``mpnet_encoder_forward`` is that forward in fp32 torch on padded batches, as ``bert_ref.bert_encoder_forward`` is
BERT's.  The float64 references follow ``encoder_kernels_ref``: ``attention_bias_ref`` (E2 with the bias table),
``embed_ln_pos_ref`` (E3 embed_ln with the position rule) and ``mpnet_stack_ref`` (the whole encoder).  Weight dicts
use the canonical names of ``ragmeup_b200.weights.weight_names`` (BERT's, plus the bias table).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from . import bert_ref
from . import encoder_kernels_ref as ekr

PAD_ID = 1
REL_BIAS = "encoder.relative_attention_bias.weight"
REL_MAX = 127                  # the kernels' table spans key - query in [-127, 127]; farther keys share its end buckets


@dataclass
class MPNetCfg(bert_ref.BertCfg):
    vocab_size: int = 30527
    max_pos: int = 514
    type_vocab: int = 1
    ln_eps: float = 1e-5
    position_mode: int = 1
    rel_buckets: int = 32


def relative_position_bucket(rel) -> np.ndarray:
    """transformers' MPNet bucket (32 buckets, max distance 128) of rel = key - query, in float64"""
    n = -np.asarray(rel, dtype=np.int64)
    ret = (n < 0).astype(np.int64) * 16
    n = np.abs(n)
    with np.errstate(divide="ignore"):
        large = 8 + (np.log(np.maximum(n, 1) / 8.0) / math.log(16.0) * 8).astype(np.int64)
    return ret + np.where(n < 8, n, np.minimum(large, 15))


def position_ids(ids: torch.Tensor) -> torch.Tensor:
    """[B, S] (or [S]) token ids -> MPNet position ids (create_position_ids_from_input_ids, padding_idx 1)"""
    m = (ids != PAD_ID).to(torch.int64)
    return torch.cumsum(m, dim=-1) * m + PAD_ID


def bias_table(bias, heads: int) -> torch.Tensor:
    """[32, heads] bias -> [heads, 2 * REL_MAX + 1] float64, entry (h, r + REL_MAX) = bias[bucket(r), h] * log2(e):
    the table the kernels index by clamp(key - query, -127, 127), in the log2 units of their scores"""
    b = ekr._f64(bias)
    buckets = torch.from_numpy(relative_position_bucket(np.arange(-REL_MAX, REL_MAX + 1))).to(b.device)
    return b[buckets].T.contiguous() * math.log2(math.e)


def mpnet_encoder_forward(w: Dict[str, object], cfg, input_ids: torch.Tensor, attention_mask: torch.Tensor,
                          matmul=None, device=None) -> torch.Tensor:
    """[B, S] ids / mask -> last hidden state [B, S, H], fp32, padded (pad with id 1, as MPNet's tokenizer does; the
    additive mask is finfo.min on padded keys, HF's eager path).  ``matmul(x, W)`` computes x @ W.T."""
    mm = matmul or (lambda x, W: x @ W.t())
    dev = device or "cpu"
    tw = lambda a: bert_ref._t(a, dev)  # noqa: E731
    input_ids, attention_mask = input_ids.to(dev), attention_mask.to(dev)
    B, S = input_ids.shape
    H, nh = cfg.hidden, cfg.heads
    dh = H // nh
    x = tw(w["embeddings.word_embeddings.weight"])[input_ids] + \
        tw(w["embeddings.position_embeddings.weight"])[position_ids(input_ids)]
    x = bert_ref._layer_norm(x, tw(w["embeddings.LayerNorm.weight"]), tw(w["embeddings.LayerNorm.bias"]), cfg.ln_eps)
    ar = torch.arange(S, device=dev)
    buckets = torch.from_numpy(relative_position_bucket((ar[None, :] - ar[:, None]).cpu().numpy())).to(dev)
    pos_bias = tw(w[REL_BIAS])[buckets].permute(2, 0, 1)[None]                 # [1, heads, S, S]
    add_mask = (1.0 - attention_mask.to(torch.float32))[:, None, None, :] * torch.finfo(torch.float32).min
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}."
        q = mm(x, tw(w[p + "attention.self.query.weight"])) + tw(w[p + "attention.self.query.bias"])
        k = mm(x, tw(w[p + "attention.self.key.weight"])) + tw(w[p + "attention.self.key.bias"])
        v = mm(x, tw(w[p + "attention.self.value.weight"])) + tw(w[p + "attention.self.value.bias"])
        q = q.view(B, S, nh, dh).transpose(1, 2)
        k = k.view(B, S, nh, dh).transpose(1, 2)
        v = v.view(B, S, nh, dh).transpose(1, 2)
        att = torch.matmul(q, k.transpose(2, 3)) / math.sqrt(dh) + pos_bias + add_mask
        att = torch.softmax(att, dim=-1)
        ctx = torch.matmul(att, v).transpose(1, 2).reshape(B, S, H)
        o = mm(ctx, tw(w[p + "attention.output.dense.weight"])) + tw(w[p + "attention.output.dense.bias"])
        x = bert_ref._layer_norm(o + x, tw(w[p + "attention.output.LayerNorm.weight"]),
                                 tw(w[p + "attention.output.LayerNorm.bias"]), cfg.ln_eps)
        f = bert_ref._gelu_erf(mm(x, tw(w[p + "intermediate.dense.weight"])) + tw(w[p + "intermediate.dense.bias"]))
        o = mm(f, tw(w[p + "output.dense.weight"])) + tw(w[p + "output.dense.bias"])
        x = bert_ref._layer_norm(o + x, tw(w[p + "output.LayerNorm.weight"]), tw(w[p + "output.LayerNorm.bias"]),
                                 cfg.ln_eps)
    return x


def st_encode(w, cfg, tokenizer, sentences: Sequence[str], pooling: str = "mean", normalize: bool = True,
              max_seq_length: int = 384, batch_size: int = 32) -> np.ndarray:
    """SentenceTransformer.encode with an MPNet model (``bert_ref.st_encode``'s batching; padding with <pad> = 1)."""
    n = len(sentences)
    if n == 0:
        return np.zeros((0, cfg.hidden), dtype=np.float32)
    order = np.argsort([-len(s) for s in sentences], kind="stable")
    out = [None] * n
    tokenizer.enable_truncation(max_length=max_seq_length, strategy="longest_first")
    tokenizer.enable_padding(pad_id=PAD_ID, pad_token="<pad>")
    with torch.no_grad():
        for s0 in range(0, n, batch_size):
            idx = order[s0:s0 + batch_size]
            enc = tokenizer.encode_batch([sentences[i].strip() for i in idx])
            ids = torch.tensor([e.ids for e in enc], dtype=torch.long)
            mask = torch.tensor([e.attention_mask for e in enc], dtype=torch.long)
            e = bert_ref.pool(mpnet_encoder_forward(w, cfg, ids, mask), mask, pooling)
            if normalize:
                e = bert_ref.l2_normalize(e)
            for j, i in enumerate(idx):
                out[i] = e[j].numpy()
    return np.asarray(out, dtype=np.float32)


def hf_embed_documents(w, cfg, tokenizer, texts: Sequence[str], **kw):
    """HuggingFaceEmbeddings.embed_documents: newline -> space, encode, .tolist()"""
    return st_encode(w, cfg, tokenizer, [t.replace("\n", " ") for t in texts], **kw).tolist()


# ------------------------------------------------------------------------------------------ float64 kernel references

def attention_bias_ref(qkv_hi, qkv_lo, cu, heads: int, table) -> tuple[torch.Tensor, torch.Tensor]:
    """E2 with the relative bias on the QKV planes [T, 3H] (q pre-scaled by log2(e) / sqrt(d_h)) of the ragged batch
    `cu`: s_ij = q_i k_j + table[h, clamp(j - i, -127, 127) + 127] (table [heads, 255] in log2 units, as the kernel
    reads it), p = 2^(s - max s), ctx = p V / sum p over the sequence's keys.  Returns (ctx [T, H], A [T, heads]) with
    A = max over the row's keys of (sum_d |q_d k_d| + |bias|), the magnitude the kernel's score rounding scales with."""
    qkv = ekr._f64(qkv_hi) + ekr._f64(qkv_lo)
    tab = ekr._f64(table).to(qkv.device)
    T, H3 = qkv.shape
    H = H3 // 3
    dh = H // heads
    ctx = torch.zeros((T, H), dtype=torch.float64, device=qkv.device)
    A = torch.zeros((T, heads), dtype=torch.float64, device=qkv.device)
    cu = [int(c) for c in cu]
    for b in range(len(cu) - 1):
        t0, t1 = cu[b], cu[b + 1]
        if t1 == t0:
            continue
        S = t1 - t0
        x = qkv[t0:t1].view(S, 3, heads, dh).transpose(0, 2)
        q, k, v = x[:, 0], x[:, 1], x[:, 2]
        ar = torch.arange(S, device=qkv.device)
        rel = (ar[None, :] - ar[:, None]).clamp(-REL_MAX, REL_MAX) + REL_MAX
        bias = tab[:, rel]                                                          # [heads, S, S]
        s = q @ k.transpose(1, 2) + bias
        p = torch.exp2(s - s.amax(2, keepdim=True))
        ctx[t0:t1] = ((p @ v) / p.sum(2, keepdim=True)).transpose(0, 1).reshape(S, H)
        A[t0:t1] = (q.abs() @ k.abs().transpose(1, 2) + bias.abs()).amax(2).T
    return ctx, A


def embed_ln_pos_ref(ids, type_ids, cu, word, pos, typ, gamma, beta, eps: float, pos_mode: int = 1):
    """E3 ``embed_ln_kernel`` with the position rule: pos_mode 0 is ``encoder_kernels_ref.embed_ln_ref``; pos_mode 1
    takes MPNet's positions per sequence (raw ids compared with 1), clamped to max_pos - 1.  Ids and type ids clamp as
    there.  Returns (y, xhat, sigma, M) as ``embed_ln_ref``."""
    if pos_mode == 0:
        return ekr.embed_ln_ref(ids, type_ids, cu, word, pos, typ, gamma, beta, eps)
    w = ekr._f64(word)
    dev = w.device
    cu_l = [int(c) for c in ekr._long(cu, dev).tolist()]
    raw = ekr._long(ids, dev)
    T = cu_l[-1]
    p = torch.zeros(T, dtype=torch.int64, device=dev)
    for b in range(len(cu_l) - 1):
        if cu_l[b + 1] > cu_l[b]:
            p[cu_l[b]:cu_l[b + 1]] = position_ids(raw[cu_l[b]:cu_l[b + 1]])
    p = p.clamp(max=int(pos.shape[0]) - 1)
    i = raw.clamp(0, int(word.shape[0]) - 1)
    ty = torch.zeros(T, dtype=torch.int64, device=dev) if type_ids is None else \
        ekr._long(type_ids, dev).clamp(0, int(typ.shape[0]) - 1)
    a, c, e = w[i], ekr._f64(typ).to(dev)[ty], ekr._f64(pos).to(dev)[p]
    y, xhat, sigma = ekr.layernorm_ref(a + c + e, gamma, beta, eps)
    return y, xhat, sigma, (a.abs() + c.abs() + e.abs()).amax(1, keepdim=True)


def mpnet_stack_ref(w, cfg, ids, cu, weights: str = "fp32", device=None) -> dict:
    """The whole MPNet encoder in float64 on the ragged batch (ids [T], cu [B + 1]), composed of the references above
    and those of ``encoder_kernels_ref`` (weights "fp32" as given, "split" as hi + lo of the split planes).  Returns
    {"hidden": [T, H], "mean" / "cls" / "mean_norm" / "cls_norm": [B, H]}, float64 on ``device``."""
    if weights not in ("fp32", "split"):
        raise ValueError(weights)
    dev = torch.device(device or "cpu")
    W = lambda name: (ekr.split_weight(w[name]) if weights == "split" else ekr._f64(w[name])).to(dev)  # noqa: E731
    V = lambda name: ekr._f64(w[name]).to(dev)                                                            # noqa: E731
    cu_l = [int(c) for c in cu]
    H, heads, eps = cfg.hidden, cfg.heads, float(cfg.ln_eps)
    x = embed_ln_pos_ref(ekr._long(ids, dev), None, ekr._long(cu_l, dev), V("embeddings.word_embeddings.weight"),
                         V("embeddings.position_embeddings.weight"), V("embeddings.token_type_embeddings.weight"),
                         V("embeddings.LayerNorm.weight"), V("embeddings.LayerNorm.bias"), eps)[0]
    tab = bias_table(V(REL_BIAS), heads)
    qs = math.log2(math.e) / math.sqrt(H // heads)
    z = torch.zeros_like
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}."
        wqkv = torch.cat([W(p + "attention.self." + n + ".weight") for n in ("query", "key", "value")])
        bqkv = torch.cat([V(p + "attention.self." + n + ".bias") for n in ("query", "key", "value")])
        qkv = ekr.gemm_ref(ekr.GEMM_BIAS_F32, x, z(x), wqkv, z(wqkv), bqkv)[0]
        qkv[:, :H] *= qs
        ctx = attention_bias_ref(qkv, z(qkv), cu_l, heads, tab)[0]
        wo = W(p + "attention.output.dense.weight")
        o = ekr.gemm_ref(ekr.GEMM_BIAS_RESID_F32, ctx, z(ctx), wo, z(wo), V(p + "attention.output.dense.bias"), x, z(x))[0]
        x1 = ekr.layernorm_ref(o, V(p + "attention.output.LayerNorm.weight"), V(p + "attention.output.LayerNorm.bias"),
                               eps)[0]
        w1 = W(p + "intermediate.dense.weight")
        f = ekr.gemm_ref(ekr.GEMM_BIAS_GELU_SPLIT, x1, z(x1), w1, z(w1), V(p + "intermediate.dense.bias"))[0]
        w2 = W(p + "output.dense.weight")
        o = ekr.gemm_ref(ekr.GEMM_BIAS_RESID_F32, f, z(f), w2, z(w2), V(p + "output.dense.bias"), x1, z(x1))[0]
        x = ekr.layernorm_ref(o, V(p + "output.LayerNorm.weight"), V(p + "output.LayerNorm.bias"), eps)[0]
    out = {"hidden": x}
    for mode, name in ((0, "mean"), (1, "cls")):
        out[name] = ekr.pool_ref(x, z(x), cu_l, mode, False)[0]
        out[name + "_norm"] = ekr.pool_ref(x, z(x), cu_l, mode, True)[0]
    return out
