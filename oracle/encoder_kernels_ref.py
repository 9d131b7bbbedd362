"""Oracle: float64 references of the encoder kernels one at a time, on the split fp16 planes they read.
TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

The encoder carries every activation and weight as two fp16 planes, v = hi + lo with hi = fp16_rn(v) and
lo = fp16_rn(v - hi) (``csrc/rmu_gemm.cuh``).  Each reference below takes the planes the kernel actually read and
evaluates hi + lo in float64 (torch, on whichever device the inputs live), so what is left between kernel and
reference is the kernel's own arithmetic:

* ``gemm_ref``: E1 ``gemm_f16x3_kernel``, sum_k (ah wh + al wh + ah wl) and the eight epilogues (BERT's bias, GELU,
  residual and q-scale; the rotary, GeGLU, fp32-residual and SwiGLU epilogues of ModernBERT, Qwen3 and Llama);
* ``attention_ref``: E2 ``attention_planes_kernel``, base-2 softmax over the keys of the same sequence;
* ``layernorm_ref``: E3 ``ln_kernel``, two-pass LayerNorm, biased variance, eps inside the square root;
* ``embed_ln_ref``: E3 ``embed_ln_kernel``, word + token-type + position rows (clamped as the kernel clamps), then
  ``layernorm_ref``;
* ``pool_ref``: E4 ``pool_kernel``, mean or CLS pooling and the optional L2 normalisation (sentence-transformers
  Pooling + Normalize);
* ``cls_head_ref``: E4 ``cls_head_kernel``, BertPooler tanh(W_p h_cls + b_p) and the classifier.

``encoder_stack_ref`` composes them into the whole encoder in float64, with the GEMM weights either as the fp32
tensors or as hi + lo of the split planes ``rmu_encoder_create`` uploads (``split_weight``).
"""
from __future__ import annotations

import math

import numpy as np
import torch

# mode ids of rmu_debug_gemm, rmu_debug_gemm_ex and rmu_debug_gemm_swiglu (include/ragmeup_b200.h)
GEMM_BIAS_F32, GEMM_BIAS_GELU_SPLIT, GEMM_BIAS_RESID_F32, GEMM_BIAS_SPLIT_QSCALE = 0, 1, 2, 3
GEMM_BIAS_SPLIT_ROPE, GEMM_BIAS_GEGLU_SPLIT, GEMM_BIAS_RESF32_F32, GEMM_BIAS_SWIGLU_SPLIT = 4, 5, 6, 7
GATED_MODES = (GEMM_BIAS_GEGLU_SPLIT, GEMM_BIAS_SWIGLU_SPLIT)


def split_f16(v) -> tuple[np.ndarray, np.ndarray]:
    """float32 v -> (hi, lo) fp16 planes as the kernels make them: hi = fp16_rn(v), lo = fp16_rn(v - hi).
    v - hi is exact in float32; below |v| ~ 0.125 lo is an fp16 subnormal."""
    v = np.asarray(v, dtype=np.float32)
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def ulp_f16(hi) -> np.ndarray:
    """float64 spacing of the fp16 grid at |hi| (2^-24 in the subnormal range); lo of a correct split is at most
    half of it"""
    _, e = np.frexp(np.asarray(hi, np.float64))          # |hi| in [2^(e-1), 2^e)
    return np.exp2(np.maximum(e - 11, -24).astype(np.float64))


def join(hi, lo) -> np.ndarray:
    """hi + lo in float64"""
    return np.asarray(hi, np.float64) + np.asarray(lo, np.float64)


def _f64(x) -> torch.Tensor:
    """planes / fp32 arrays (numpy or torch, any device) -> float64 torch tensor on the same device"""
    return x.to(torch.float64) if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x, np.float64))


def deblock(t) -> torch.Tensor:
    """[..., N] in the gated modes' column order (128-column blocks of 64 input | 64 gate columns) -> [..., N] with
    every input column first, then every gate column (in | gate of the natural [2F] layout)"""
    t = _f64(t)
    blk = t.reshape(*t.shape[:-1], t.shape[-1] // 128, 2, 64)
    return torch.cat([blk[..., 0, :].flatten(-2), blk[..., 1, :].flatten(-2)], -1)


def rope_partner(t, qcols: int, head_dim: int) -> torch.Tensor:
    """[M, N] -> the value at each column's rotation partner (c <-> c + d/2 within a head) for the q and k columns
    (col < 2 qcols); v columns map to themselves"""
    t = _f64(t)
    n = 2 * qcols
    h = t[:, :n].reshape(t.shape[0], n // head_dim, 2, head_dim // 2)
    return torch.cat([h.flip(2).reshape(t.shape[0], n), t[:, n:]], 1)


def rope_columns(pos, rope_cos, rope_sin, N: int, qcols: int, head_dim: int) -> tuple[torch.Tensor, torch.Tensor]:
    """(C, Sn) [M, N] float64 of the rotary epilogue: out_c = x_c C_c + x_partner(c) Sn_c, from the float32 tables at
    each row's position clamped into [0, rope_rows) as the kernel clamps it.  Sn = -sin on the first half of a head,
    +sin on the second; C = 1 and Sn = 0 on the v columns."""
    c, s = _f64(rope_cos), _f64(rope_sin)
    p = _long(pos, c.device).clamp(0, int(c.shape[0]) - 1)
    M, n = int(p.shape[0]), 2 * qcols
    cp, sp = c[p], s[p]                                       # [M, head_dim / 2]
    C = torch.ones((M, N), dtype=torch.float64, device=c.device)
    Sn = torch.zeros_like(C)
    C[:, :n] = torch.cat([cp, cp], 1).repeat(1, n // head_dim)
    Sn[:, :n] = torch.cat([-sp, sp], 1).repeat(1, n // head_dim)
    return C, Sn


def gemm_ref(mode: int, a_hi, a_lo, w_hi, w_lo, bias, res_hi=None, res_lo=None, qcols: int = 0,
             qscale: float = 1.0, res_f32=None, pos=None, rope_cos=None, rope_sin=None,
             head_dim: int = 64) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """E1 on A [M, K] and W [N, K] planes.  Returns (out, x, S): out [M, N] float64 after the epilogue of `mode`,
    x = the pre-epilogue sum + bias (GELU's argument), and S_ij = sum_k |a_ik w_jk| for the error bound.

    * mode 4 (rotary): q | k columns (col < 2 qcols) rotated per head of head_dim at pos[row] (``rope_columns``), then
      q (col < qcols) times float32(qscale); v as mode 3 leaves it.  x and S are before the rotation: the partner
      column's are ``rope_partner(x / S, qcols, head_dim)``.
    * modes 5 (GeGLU) and 7 (SwiGLU): W in the kernel's 128-row blocks of 64 input | 64 gate rows; out [M, N / 2] =
      act(in) * gate with act = gelu_erf / silu, in natural column order.  x and S are ``deblock``-ed: columns
      [0, N / 2) are the inputs', [N / 2, N) the gates'.
    * mode 6: out = x + res_f32 (fp32 [M, N])."""
    ah, al, wh, wl = _f64(a_hi), _f64(a_lo), _f64(w_hi), _f64(w_lo)
    acc = ah @ wh.T + al @ wh.T + ah @ wl.T          # the three products the kernel issues (no lo * lo)
    S = (ah + al).abs() @ (wh + wl).abs().T
    x = acc + _f64(bias).to(acc.device)[None, :]
    if mode in GATED_MODES:
        x, S = deblock(x), deblock(S)
        F = x.shape[1] // 2
        xin, gate = x[:, :F], x[:, F:]
        act = 0.5 * xin * (1.0 + torch.special.erf(xin / math.sqrt(2.0))) if mode == GEMM_BIAS_GEGLU_SPLIT \
            else xin * torch.sigmoid(xin)
        return act * gate, x, S
    if mode == GEMM_BIAS_SPLIT_ROPE:
        C, Sn = rope_columns(pos, rope_cos, rope_sin, x.shape[1], qcols, head_dim)
        out = x * C.to(x.device) + rope_partner(x, qcols, head_dim) * Sn.to(x.device)
        out[:, :qcols] *= float(np.float32(qscale))
        return out, x, S
    if mode == GEMM_BIAS_RESF32_F32:
        return x + _f64(res_f32).to(x.device), x, S
    if mode == GEMM_BIAS_F32:
        out = x
    elif mode == GEMM_BIAS_GELU_SPLIT:
        out = 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))
    elif mode == GEMM_BIAS_RESID_F32:
        out = x + (_f64(res_hi) + _f64(res_lo))
    elif mode == GEMM_BIAS_SPLIT_QSCALE:
        sc = torch.ones(x.shape[1], dtype=torch.float64, device=x.device)
        sc[:qcols] = float(np.float32(qscale))
        out = x * sc[None, :]
    else:
        raise ValueError(mode)
    return out, x, S


def attention_ref(qkv_hi, qkv_lo, cu, heads: int) -> tuple[torch.Tensor, torch.Tensor]:
    """E2 on the QKV planes [T, 3H] (q | k | v, q pre-scaled by log2(e) / sqrt(d_h)) of the ragged batch `cu`.
    Per sequence and head: s = q k^T, p = 2^(s - max s), ctx = p V / sum p, over that sequence's keys only.
    Returns (ctx [T, H], A [T, heads]) with A = max over the row's keys of sum_d |q_d k_d|, the magnitude the
    kernel's score rounding scales with."""
    qkv = _f64(qkv_hi) + _f64(qkv_lo)
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
        x = qkv[t0:t1].view(t1 - t0, 3, heads, dh).transpose(0, 2)      # [heads, 3, S, dh]
        q, k, v = x[:, 0], x[:, 1], x[:, 2]
        s = q @ k.transpose(1, 2)
        p = torch.exp2(s - s.amax(2, keepdim=True))
        ctx[t0:t1] = ((p @ v) / p.sum(2, keepdim=True)).transpose(0, 1).reshape(t1 - t0, H)
        A[t0:t1] = (q.abs() @ k.abs().transpose(1, 2)).amax(2).T
    return ctx, A


def layernorm_ref(x, gamma, beta, eps: float) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """E3 on fp32 rows x [T, H]: two-pass mean / biased variance in float64, eps (as the fp32 the kernel gets) inside
    the square root.  Returns (y, xhat, sigma) with sigma = sqrt(var + eps) per row."""
    x = _f64(x)
    mu = x.mean(1, keepdim=True)
    var = ((x - mu) ** 2).mean(1, keepdim=True)
    sigma = torch.sqrt(var + float(np.float32(eps)))
    xhat = (x - mu) / sigma
    return xhat * _f64(gamma)[None, :] + _f64(beta)[None, :], xhat, sigma


def _long(x, device) -> torch.Tensor:
    return (x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x))).to(device=device, dtype=torch.int64)


def embed_ln_ref(ids, type_ids, cu, word, pos, typ, gamma, beta, eps: float):
    """E3 ``embed_ln_kernel`` on the fp32 tables word [vocab, H], pos [max_pos, H], typ [type_vocab, H] for the ragged
    batch `cu` (type_ids None = all 0).  Token ids are clamped into [0, vocab), type ids into [0, type_vocab) and
    positions (the token's offset in its sequence) to max_pos - 1, as the kernel does.  x = word + typ + pos in float64,
    then ``layernorm_ref``.  Returns (y, xhat, sigma, M) with M [T, 1] = max_d (|word_d| + |typ_d| + |pos_d|), the
    magnitude the kernel's fp32 three-term sum rounds against."""
    w = _f64(word)
    dev = w.device
    cu = _long(cu, dev)
    T = int(cu[-1])
    lens = cu[1:] - cu[:-1]
    p = torch.arange(T, device=dev) - torch.repeat_interleave(cu[:-1], lens)
    p = p.clamp(max=int(pos.shape[0]) - 1)
    i = _long(ids, dev).clamp(0, int(word.shape[0]) - 1)
    ty = torch.zeros(T, dtype=torch.int64, device=dev) if type_ids is None else \
        _long(type_ids, dev).clamp(0, int(typ.shape[0]) - 1)
    a, c, e = w[i], _f64(typ).to(dev)[ty], _f64(pos).to(dev)[p]
    y, xhat, sigma = layernorm_ref(a + c + e, gamma, beta, eps)
    return y, xhat, sigma, (a.abs() + c.abs() + e.abs()).amax(1, keepdim=True)


def pool_ref(hi, lo, cu, mode: int, normalize: bool):
    """E4 ``pool_kernel`` on planes [T, H] of the ragged batch `cu`: mode 0 = mean (sum / max(S, 1e-9), so an empty
    sequence gives 0), mode 1 = CLS (row cu[b], 0 for an empty sequence); then x / max(||x||, 1e-12) when normalize.
    Only rows the kernel reads are read.  Returns (out [B, H], m [B, H] before normalisation, P [B, H]) with
    P = sum over the sequence of |x_td| (mean) or 0 (CLS, an exact copy): the magnitude the fp32 sum rounds against."""
    x = _f64(hi) + _f64(lo)
    cu = [int(c) for c in cu]
    B, H = len(cu) - 1, x.shape[1]
    m = torch.zeros((B, H), dtype=torch.float64, device=x.device)
    P = torch.zeros_like(m)
    for b in range(B):
        t0, t1 = cu[b], cu[b + 1]
        if t1 == t0:
            continue
        if mode == 1:
            m[b] = x[t0]
        else:
            m[b] = x[t0:t1].sum(0) / (t1 - t0)
            P[b] = x[t0:t1].abs().sum(0)
    out = m / m.norm(dim=1, keepdim=True).clamp(min=1e-12) if normalize else m
    return out, m, P


def cls_head_ref(hi, lo, cu, pw, pb, cw, cb):
    """E4 ``cls_head_kernel`` on planes [T, H] of the ragged batch `cu`: h = row cu[b] (0 for an empty sequence),
    z = pw h + pb, pooled = tanh(z), logits = cw pooled + cb, in float64.  Returns (logits [B, L], z [B, H], pooled,
    A [B, H], C [B, L]) with A_bj = sum_d |pw_jd h_d| and C_bc = sum_j |cw_cj pooled_j|, the magnitudes the two dot
    products round against."""
    x = _f64(hi) + _f64(lo)
    cu = [int(c) for c in cu]
    B, H = len(cu) - 1, x.shape[1]
    h = torch.zeros((B, H), dtype=torch.float64, device=x.device)
    for b in range(B):
        if cu[b + 1] > cu[b]:
            h[b] = x[cu[b]]
    W, Wc = _f64(pw).to(x.device), _f64(cw).to(x.device)
    z = h @ W.T + _f64(pb).to(x.device)[None, :]
    pooled = torch.tanh(z)
    logits = pooled @ Wc.T + _f64(cb).to(x.device)[None, :]
    return logits, z, pooled, h.abs() @ W.abs().T, pooled.abs() @ Wc.abs().T


# the six GEMM weights of a layer, which rmu_encoder_create uploads as split planes
GEMM_WEIGHTS = ("attention.self.query.weight", "attention.self.key.weight", "attention.self.value.weight",
                "attention.output.dense.weight", "intermediate.dense.weight", "output.dense.weight")


def split_weight(w) -> torch.Tensor:
    """fp32 weight (numpy or torch, any device) -> hi + lo of its split planes in float64, on the same device.  For
    |w| < 2^-14 * 2^11 ~ 0.125 the lo plane is an fp16 subnormal, so a weight keeps max(2^-22 |w|, 2^-25) of error
    instead of 2^-22 |w|."""
    t = (w if isinstance(w, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(w, np.float32))).to(torch.float32)
    hi = t.half()
    return hi.double() + (t - hi.float()).half().double()


def encoder_stack_ref(w, cfg, ids, type_ids, cu, weights: str = "fp32", device=None) -> dict:
    """The whole encoder in float64 on the ragged batch (ids [T], type_ids [T] or None = all 0, cu [B + 1]), with the
    kernels' documented rules: ids, type ids and positions clamped (``embed_ln_ref``), an empty sequence embeds as
    zeros and scores W_c tanh(b_p) + b_c (``pool_ref``, ``cls_head_ref``).  ``w`` is the weight dict of
    ``ragmeup_b200.weights.weight_names``; cfg anything with hidden, heads, layers and ln_eps.  weights = "fp32" takes the
    GEMM weights as given, "split" as hi + lo of their split planes (``split_weight``).  Runs in torch on ``device``
    (default the CPU).  Returns {"hidden": [T, H], "mean" / "cls" / "mean_norm" / "cls_norm": [B, H], and "logits":
    [B, num_labels] when w holds the head}, float64 on ``device``."""
    if weights not in ("fp32", "split"):
        raise ValueError(weights)
    dev = torch.device(device or "cpu")
    W = lambda name: (split_weight(w[name]) if weights == "split" else _f64(w[name])).to(dev)  # noqa: E731
    V = lambda name: _f64(w[name]).to(dev)                                                        # noqa: E731
    cu_l = [int(c) for c in cu]
    H, heads, eps = cfg.hidden, cfg.heads, float(cfg.ln_eps)
    x = embed_ln_ref(_long(ids, dev), None if type_ids is None else _long(type_ids, dev), _long(cu_l, dev),
                     V("embeddings.word_embeddings.weight"), V("embeddings.position_embeddings.weight"),
                     V("embeddings.token_type_embeddings.weight"), V("embeddings.LayerNorm.weight"),
                     V("embeddings.LayerNorm.bias"), eps)[0]
    qs = math.log2(math.e) / math.sqrt(H // heads)        # the exact scale attention_ref's base-2 softmax expects
    z = torch.zeros_like
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}."
        wqkv = torch.cat([W(p + "attention.self." + n + ".weight") for n in ("query", "key", "value")])
        bqkv = torch.cat([V(p + "attention.self." + n + ".bias") for n in ("query", "key", "value")])
        qkv = gemm_ref(GEMM_BIAS_F32, x, z(x), wqkv, z(wqkv), bqkv)[0]
        qkv[:, :H] *= qs
        ctx = attention_ref(qkv, z(qkv), cu_l, heads)[0]
        wo = W(p + "attention.output.dense.weight")
        o = gemm_ref(GEMM_BIAS_RESID_F32, ctx, z(ctx), wo, z(wo), V(p + "attention.output.dense.bias"), x, z(x))[0]
        x1 = layernorm_ref(o, V(p + "attention.output.LayerNorm.weight"), V(p + "attention.output.LayerNorm.bias"), eps)[0]
        w1 = W(p + "intermediate.dense.weight")
        f = gemm_ref(GEMM_BIAS_GELU_SPLIT, x1, z(x1), w1, z(w1), V(p + "intermediate.dense.bias"))[0]
        w2 = W(p + "output.dense.weight")
        o = gemm_ref(GEMM_BIAS_RESID_F32, f, z(f), w2, z(w2), V(p + "output.dense.bias"), x1, z(x1))[0]
        x = layernorm_ref(o, V(p + "output.LayerNorm.weight"), V(p + "output.LayerNorm.bias"), eps)[0]
    out = {"hidden": x}
    for mode, name in ((0, "mean"), (1, "cls")):
        out[name] = pool_ref(x, z(x), cu_l, mode, False)[0]
        out[name + "_norm"] = pool_ref(x, z(x), cu_l, mode, True)[0]
    if "pooler.dense.weight" in w:
        out["logits"] = cls_head_ref(x, z(x), cu_l, V("pooler.dense.weight"), V("pooler.dense.bias"),
                                     V("classifier.weight"), V("classifier.bias"))[0]
    return out
