"""Qwen3 run as an encoder (transformers 5.5 ``Qwen3Model``), in float64 or float32, over the canonical weights of
``ragmeup_b200.weights.qwen3_weight_names``; plus its output rows and the reranker's pair assembly.

One sequence at a time, positions 0..S-1, causal attention, so no padding or mask enters the arithmetic.  The rotary
cos / sin come from the float32 tables ``weights.rope_table`` builds, as in the model; everything else runs in the
requested dtype.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np
import torch

from ragmeup_b200.weights import Qwen3Config, rope_table


def _rms(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def weights(w: Dict[str, np.ndarray], dtype=torch.float64, device="cpu") -> Dict[str, torch.Tensor]:
    """the canonical arrays as tensors of ``dtype`` on ``device`` (convert once for many ``hidden`` calls)"""
    return {k: torch.as_tensor(np.asarray(v)).to(device=device, dtype=dtype) for k, v in w.items()}


def hidden(w, cfg: Qwen3Config, ids: Sequence[int], dtype=torch.float64) -> torch.Tensor:
    """final hidden state (after ``norm``) of one sequence -> [S, H]; ``w`` holds numpy arrays or tensors (their
    device is used)"""
    W = {k: torch.as_tensor(v).to(dtype) for k, v in w.items()}
    dev = W["norm.weight"].device
    d, nh, kv, eps = cfg.head_dim, cfg.heads, cfg.kv_heads, cfg.ln_eps
    S = len(ids)
    cos_t, sin_t = (torch.from_numpy(t[:S]).to(device=dev, dtype=dtype) for t in rope_table(cfg.rope_theta, d, cfg.max_pos))
    cos, sin = torch.cat([cos_t, cos_t], -1)[:, None, :], torch.cat([sin_t, sin_t], -1)[:, None, :]

    def rope(x):
        rot = torch.cat([-x[..., d // 2:], x[..., :d // 2]], -1)
        return x * cos + rot * sin

    h = W["embed_tokens.weight"][torch.as_tensor(list(ids), dtype=torch.long, device=dev)]
    mask = torch.ones(S, S, dtype=torch.bool, device=dev).tril()
    for l in range(cfg.layers):
        p = f"layers.{l}."
        x = _rms(h, W[p + "input_layernorm.weight"], eps)
        q = (x @ W[p + "self_attn.q_proj.weight"].T).view(S, nh, d)
        k = (x @ W[p + "self_attn.k_proj.weight"].T).view(S, kv, d)
        v = (x @ W[p + "self_attn.v_proj.weight"].T).view(S, kv, d)
        q = rope(_rms(q, W[p + "self_attn.q_norm.weight"], eps))
        k = rope(_rms(k, W[p + "self_attn.k_norm.weight"], eps))
        g = nh // kv
        k, v = k.repeat_interleave(g, 1), v.repeat_interleave(g, 1)
        s = torch.einsum("ihd,jhd->hij", q, k) * d ** -0.5
        s = s.masked_fill(~mask, float("-inf")).softmax(-1)
        ctx = torch.einsum("hij,jhd->ihd", s, v).reshape(S, nh * d)
        h = h + ctx @ W[p + "self_attn.o_proj.weight"].T
        x2 = _rms(h, W[p + "post_attention_layernorm.weight"], eps)
        gate, up = x2 @ W[p + "mlp.gate_proj.weight"].T, x2 @ W[p + "mlp.up_proj.weight"].T
        h = h + (torch.nn.functional.silu(gate) * up) @ W[p + "mlp.down_proj.weight"].T
    return _rms(h, W["norm.weight"], eps)


def head_row(ids: Sequence[int], pad_id: int) -> int:
    """transformers' last_non_pad_token: the rightmost index whose id != pad_id (0 when there is none); pad_id < 0:
    the last index"""
    if pad_id < 0:
        return len(ids) - 1
    keep = [i for i, t in enumerate(ids) if t != pad_id]
    return keep[-1] if keep else 0


def embed(w, cfg: Qwen3Config, seqs: List[Sequence[int]], normalize: bool, dtype=torch.float64) -> torch.Tensor:
    """last-token embeddings [B, H] (sentence-transformers' lasttoken pooling, then Normalize when asked)"""
    rows = torch.stack([hidden(w, cfg, s, dtype)[-1] for s in seqs])
    return torch.nn.functional.normalize(rows, dim=-1) if normalize else rows


def logits(w, cfg: Qwen3Config, seqs: List[Sequence[int]], pad_id: int, dtype=torch.float64) -> torch.Tensor:
    """the last-token head [B, num_labels]: head . hidden[head_row]"""
    Wh = torch.as_tensor(w["head"]).to(dtype)
    return torch.stack([hidden(w, cfg, s, dtype)[head_row(s, pad_id)] @ Wh.T for s in seqs])


def yes_probability(no_yes: torch.Tensor) -> torch.Tensor:
    """[B, 2] (no, yes) logits -> exp(log_softmax(.)[:, 1]), as the Qwen3-Reranker model card scores"""
    return no_yes.log_softmax(1)[:, 1].exp()


def rerank_ids(tok, prefix: str, suffix: str, instruction: str, pairs, max_length: int) -> List[List[int]]:
    """the model card's process_inputs through a transformers tokenizer ``tok``: each formatted text tokenised with
    truncation to max_length - len(prefix) - len(suffix), between the prefix and suffix tokens"""
    pre = tok.encode(prefix, add_special_tokens=False)
    suf = tok.encode(suffix, add_special_tokens=False)
    texts = [f"<Instruct>: {instruction}\n<Query>: {q}\n<Document>: {d}" for q, d in pairs]
    enc = tok(texts, padding=False, truncation="longest_first", return_attention_mask=False,
              max_length=max_length - len(pre) - len(suf))
    return [pre + e + suf for e in enc["input_ids"]]
