"""Oracle: ColBERT late-interaction scoring, restated in fp32 torch, and float64 references of its device parts.
TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

[3P-recall: colbert-ai 0.2.x (``QueryTokenizer.tensorize``, ``DocTokenizer.tensorize``, ``ColBERT.query``,
``ColBERT.doc``, ``colbert_score``), not installed here; restated from memory]

* Query: ``tok([". " + q], padding="max_length", truncation=True, max_length=query_maxlen)``; ``ids[:, 1]`` = the
  query marker ([unused0]); ``ids[ids == pad_id] = mask_id``; with ``attend_to_mask_tokens = False`` the attention
  mask stays the tokenizer's (0 on the [MASK] padding), so those rows are queries but not keys.  Every row is kept.
* Document: ``tok([". " + d], padding="longest", truncation="longest_first", max_length=doc_maxlen)``; ``ids[:, 1]`` =
  the document marker ([unused1]); the score mask is ``id not in skiplist and id != pad_id``, the skiplist being the
  first id of each ``string.punctuation`` character (``mask_punctuation``).
* Vectors: ``F.normalize(linear(bert(ids, attention_mask)[0]), p=2, dim=2)`` (no bias, eps 1e-12); BERT gets no token
  types.
* ``colbert_score``: the scores ``D @ Q.T`` of masked document rows are set to -9999 (``colbert_score_reduce``), then
  ``.max(1).values.sum(-1)``.

The tokenisation here uses HF ``tokenizers``' own truncation and padding, not the product's code.
"""
from __future__ import annotations

import math
import string
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch
from tokenizers import Tokenizer

from . import bert_ref
from . import encoder_kernels_ref as ekr


def _copy(tok: Tokenizer) -> Tokenizer:
    return Tokenizer.from_str(tok.to_str())


def skiplist(tok: Tokenizer) -> List[int]:
    out = []
    for c in string.punctuation:
        ids = tok.encode(c, add_special_tokens=False).ids
        if ids:
            out.append(ids[0])
    return sorted(set(out))


def tokenize_queries(tok: Tokenizer, spec, texts: Sequence[str]) -> Tuple[torch.Tensor, torch.Tensor]:
    """-> (ids [n, query_maxlen], attention_mask [n, query_maxlen]) int64"""
    t = _copy(tok)
    pad, mask = t.token_to_id("[PAD]"), t.token_to_id("[MASK]")
    t.enable_truncation(max_length=spec.query_maxlen)
    t.enable_padding(pad_id=pad, pad_token="[PAD]", length=spec.query_maxlen)
    enc = t.encode_batch([". " + x for x in texts])
    ids = torch.tensor([e.ids for e in enc], dtype=torch.long)
    am = torch.tensor([e.attention_mask for e in enc], dtype=torch.long)
    ids[:, 1] = t.token_to_id(spec.query_token)
    ids[ids == pad] = mask
    return ids, am


def tokenize_docs(tok: Tokenizer, spec, texts: Sequence[str]) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """-> (ids [n, S], attention_mask [n, S], score mask [n, S]) with S the longest document"""
    t = _copy(tok)
    pad = t.token_to_id("[PAD]")
    t.enable_truncation(max_length=spec.doc_maxlen, strategy="longest_first")
    t.enable_padding(pad_id=pad, pad_token="[PAD]")
    enc = t.encode_batch([". " + x for x in texts])
    ids = torch.tensor([e.ids for e in enc], dtype=torch.long)
    am = torch.tensor([e.attention_mask for e in enc], dtype=torch.long)
    ids[:, 1] = t.token_to_id(spec.doc_token)
    skip = set(skiplist(t)) if spec.mask_punctuation else set()
    keep = torch.tensor([[(x not in skip) and (x != pad) for x in row] for row in ids.tolist()], dtype=torch.bool)
    return ids, am, keep


def vectors(w, cfg, linear, ids: torch.Tensor, attention_mask: torch.Tensor, device=None) -> torch.Tensor:
    """fp32 forward -> normalize(linear(h)) [n, S, dim]"""
    with torch.no_grad():
        h = bert_ref.bert_encoder_forward(w, cfg, ids, attention_mask, None, device=device)
        lin = bert_ref._t(linear, h.device)
        return torch.nn.functional.normalize(h @ lin.T, p=2, dim=2)


def colbert_score(Q: torch.Tensor, D: torch.Tensor, D_mask: torch.Tensor) -> torch.Tensor:
    """Q [Lq, dim] against documents D [n, S, dim] with score mask [n, S] -> [n]"""
    scores = D @ Q.T                                          # [n, S, Lq]
    scores[~D_mask.to(D.device)] = -9999                      # colbert_score_reduce: masked document rows never win
    return scores.max(1).values.sum(-1)


def score_pairs(w, cfg, linear, spec, tok: Tokenizer, pairs: Sequence[Tuple[str, str]], device=None) -> np.ndarray:
    """HuggingFaceCrossEncoder.score on a ColBERT checkpoint: the MaxSim score of every (query, document) pair,
    float32 [n]"""
    if len(pairs) == 0:
        raise IndexError("score_pairs: empty input")
    queries = list(dict.fromkeys(p[0] for p in pairs))
    docs = list(dict.fromkeys(p[1] for p in pairs))
    qi, am = tokenize_queries(tok, spec, queries)
    Q = vectors(w, cfg, linear, qi, am, device)
    out = np.empty(len(pairs), np.float32)
    D_all = {}
    for s in range(0, len(docs), 32):
        chunk = docs[s:s + 32]
        di, dam, keep = tokenize_docs(tok, spec, chunk)
        D = vectors(w, cfg, linear, di, dam, device)
        for j, d in enumerate(chunk):
            D_all[d] = (D[j:j + 1], keep[j:j + 1])
    qpos = {q: i for i, q in enumerate(queries)}
    for n, (q, d) in enumerate(pairs):
        D, keep = D_all[d]
        out[n] = float(colbert_score(Q[qpos[q]], D, keep)[0])
    return out


# --------------------------------------------------------------------------------------------- float64 references
def attention_keys_ref(qkv_hi, qkv_lo, cu, nkeys, heads: int):
    """E2 with a key limit on the QKV planes [T, 3H] (q pre-scaled by log2(e) / sqrt(d_h)): sequence b's rows are all
    queries, its keys are rows 0 .. min(max(nkeys[b], 1), S_b) - 1.  ``encoder_kernels_ref.attention_ref`` on the
    sequence's query rows against its key rows, float64.  Returns (ctx [T, H], A [T, heads])."""
    qkv = ekr._f64(qkv_hi) + ekr._f64(qkv_lo)
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
        nk = min(max(int(nkeys[b]), 1), t1 - t0)
        x = qkv[t0:t1].view(t1 - t0, 3, heads, dh).transpose(0, 2)      # [heads, 3, S, dh]
        q, k, v = x[:, 0], x[:, 1, :nk], x[:, 2, :nk]
        s = q @ k.transpose(1, 2)
        p = torch.exp2(s - s.amax(2, keepdim=True))
        ctx[t0:t1] = ((p @ v) / p.sum(2, keepdim=True)).transpose(0, 1).reshape(t1 - t0, H)
        A[t0:t1] = (q.abs() @ k.abs().transpose(1, 2)).amax(2).T
    return ctx, A


def colbert_stack_ref(w, cfg, linear, ids, cu, nkeys=None, keep=None, weights: str = "split", device=None) -> Dict:
    """``encoder_kernels_ref.encoder_stack_ref``'s float64 forward with the key limit in every layer, then the
    projection (``linear`` as hi + lo of its split planes with weights = "split") and the normalisation; tokens with
    keep 0 get zero vectors.  Returns {"hidden": [T, H], "proj": [T, dim], "vectors": [T, dim]} float64."""
    dev = torch.device(device or "cpu")
    W = lambda name: (ekr.split_weight(w[name]) if weights == "split" else ekr._f64(w[name])).to(dev)  # noqa: E731
    V = lambda name: ekr._f64(w[name]).to(dev)                                                          # noqa: E731
    cu_l = [int(c) for c in cu]
    nk = [c1 - c0 for c0, c1 in zip(cu_l[:-1], cu_l[1:])] if nkeys is None else [int(n) for n in nkeys]
    H, heads, eps = cfg.hidden, cfg.heads, float(cfg.ln_eps)
    x = ekr.embed_ln_ref(ekr._long(ids, dev), None, ekr._long(cu_l, dev), V("embeddings.word_embeddings.weight"),
                         V("embeddings.position_embeddings.weight"), V("embeddings.token_type_embeddings.weight"),
                         V("embeddings.LayerNorm.weight"), V("embeddings.LayerNorm.bias"), eps)[0]
    qs = math.log2(math.e) / math.sqrt(H // heads)
    z = torch.zeros_like
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}."
        wqkv = torch.cat([W(p + "attention.self." + n + ".weight") for n in ("query", "key", "value")])
        bqkv = torch.cat([V(p + "attention.self." + n + ".bias") for n in ("query", "key", "value")])
        qkv = ekr.gemm_ref(ekr.GEMM_BIAS_F32, x, z(x), wqkv, z(wqkv), bqkv)[0]
        qkv[:, :H] *= qs
        ctx = attention_keys_ref(qkv, z(qkv), cu_l, nk, heads)[0]
        wo = W(p + "attention.output.dense.weight")
        o = ekr.gemm_ref(ekr.GEMM_BIAS_RESID_F32, ctx, z(ctx), wo, z(wo), V(p + "attention.output.dense.bias"), x, z(x))[0]
        x1 = ekr.layernorm_ref(o, V(p + "attention.output.LayerNorm.weight"), V(p + "attention.output.LayerNorm.bias"),
                               eps)[0]
        w1 = W(p + "intermediate.dense.weight")
        f = ekr.gemm_ref(ekr.GEMM_BIAS_GELU_SPLIT, x1, z(x1), w1, z(w1), V(p + "intermediate.dense.bias"))[0]
        w2 = W(p + "output.dense.weight")
        o = ekr.gemm_ref(ekr.GEMM_BIAS_RESID_F32, f, z(f), w2, z(w2), V(p + "output.dense.bias"), x1, z(x1))[0]
        x = ekr.layernorm_ref(o, V(p + "output.LayerNorm.weight"), V(p + "output.LayerNorm.bias"), eps)[0]
    lin = (ekr.split_weight(linear) if weights == "split" else ekr._f64(linear)).to(dev)
    proj = x @ lin.T
    vec = proj / proj.norm(dim=1, keepdim=True).clamp(min=1e-12)
    if keep is not None:
        vec = vec * torch.as_tensor(np.asarray(keep) != 0, device=dev)[:, None]
    return {"hidden": x, "proj": proj, "vectors": vec}


def maxsim_fsum(q, q_cu, d, d_cu, keep, pair_q, pair_d) -> np.ndarray:
    """MaxSim replayed in float64 with ``math.fsum``: for each pair, fsum over the query's tokens of the max over the
    document's kept tokens of fsum_c q_c d_c, on the given (fp32) vectors.  Returns (score [n], M [n]) with M = the
    fsum over query tokens of max_j sum_c |q_c d_c|, the magnitude an fp32 evaluation rounds against."""
    q, d = np.asarray(q, np.float64), np.asarray(d, np.float64)
    out, mag = np.empty(len(pair_q)), np.empty(len(pair_q))
    for n, (a, b) in enumerate(zip(pair_q, pair_d)):
        Q = q[q_cu[a]:q_cu[a + 1]]
        rows = [j for j in range(d_cu[b], d_cu[b + 1]) if keep is None or keep[j]]
        D = d[rows]
        best = [max(math.fsum(qi * dj) for dj in D) for qi in Q]
        out[n] = math.fsum(best)
        mag[n] = math.fsum(float(np.max(np.abs(D) @ np.abs(qi))) for qi in Q)
    return out, mag
