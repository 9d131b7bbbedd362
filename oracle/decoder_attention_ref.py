"""Oracle for attention provenance (``server/provenance.py:19-98``, ``compute_attention``).  TEST INFRASTRUCTURE ONLY
(see ``oracle/__init__.py``).

* ``last_attention``: the last layer's attention probabilities [heads, S, S] of one sequence through a Qwen3 or Llama
  decoder (transformers' eager ``attentions[-1][0]``), in float64 or float32.  It is ``qwen3_ref.hidden``'s forward,
  with the per-head q / k RMSNorm optional (``qk_norm=False`` is Llama) and the rope table of the config (``llama3``
  scaling for a ``LlamaConfig``); ``hidden`` returns the final hidden state of the same forward.
* ``attention_scores``: the reference's span arithmetic over a given attention tensor A [heads, T, T].  Each part
  (query, answer, each document) is located at its first occurrence in the thread's tokens; its block is the slice
  [start : start + len - 1] (the reference leaves the part's last token out), and an empty part is found at 0, giving
  the slice [0 : -1].  A block's value is the mean of A over every head and the block's rows and columns (NaN when
  empty).  qq, qa, aa and aq always enter the total; each document adds ad and da, and qd and dq unless
  attribute_include_query == "False"; every value enters only when > 0.  A document scores the mean of its kept values
  (NaN if none) over the mean of all kept values.
PARITY STATUS: the forward is checked against transformers' LlamaForCausalLM and Qwen3ForCausalLM in float64
(tests/test_attention_provenance_cpu.py); the span arithmetic is restated from the reference's code and checked on
hand-built tensors.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
import torch

from oracle.qwen3_ref import _rms
from ragmeup_b200.weights import rope_table


def _forward(w, cfg, ids: Sequence[int], dtype, qk_norm: bool, probs: bool) -> torch.Tensor:
    W = {k: torch.as_tensor(v).to(dtype) for k, v in w.items()}
    dev = W["norm.weight"].device
    d, nh, kv, eps = cfg.head_dim, cfg.heads, cfg.kv_heads, cfg.ln_eps
    S = len(ids)
    table = rope_table(cfg.rope_theta, d, cfg.max_pos, getattr(cfg, "rope_scaling", None))
    cos_t, sin_t = (torch.from_numpy(t[:S]).to(device=dev, dtype=dtype) for t in table)
    cos, sin = torch.cat([cos_t, cos_t], -1)[:, None, :], torch.cat([sin_t, sin_t], -1)[:, None, :]

    def rope(x):
        return x * cos + torch.cat([-x[..., d // 2:], x[..., :d // 2]], -1) * sin

    h = W["embed_tokens.weight"][torch.as_tensor(list(ids), dtype=torch.long, device=dev)]
    mask = torch.ones(S, S, dtype=torch.bool, device=dev).tril()
    for l in range(cfg.layers):
        p = f"layers.{l}."
        x = _rms(h, W[p + "input_layernorm.weight"], eps)
        q = (x @ W[p + "self_attn.q_proj.weight"].T).view(S, nh, d)
        k = (x @ W[p + "self_attn.k_proj.weight"].T).view(S, kv, d)
        v = (x @ W[p + "self_attn.v_proj.weight"].T).view(S, kv, d)
        if qk_norm:
            q, k = _rms(q, W[p + "self_attn.q_norm.weight"], eps), _rms(k, W[p + "self_attn.k_norm.weight"], eps)
        q, k = rope(q), rope(k)
        g = nh // kv
        k, v = k.repeat_interleave(g, 1), v.repeat_interleave(g, 1)
        s = torch.einsum("ihd,jhd->hij", q, k) * d ** -0.5
        s = s.masked_fill(~mask, float("-inf")).softmax(-1)
        if probs and l == cfg.layers - 1:
            return s
        h = h + torch.einsum("hij,jhd->ihd", s, v).reshape(S, nh * d) @ W[p + "self_attn.o_proj.weight"].T
        x2 = _rms(h, W[p + "post_attention_layernorm.weight"], eps)
        gate, up = x2 @ W[p + "mlp.gate_proj.weight"].T, x2 @ W[p + "mlp.up_proj.weight"].T
        h = h + (torch.nn.functional.silu(gate) * up) @ W[p + "mlp.down_proj.weight"].T
    return _rms(h, W["norm.weight"], eps)


def hidden(w, cfg, ids: Sequence[int], dtype=torch.float64, qk_norm: bool = True) -> torch.Tensor:
    """final hidden state (after ``norm``) of one sequence -> [S, H]"""
    return _forward(w, cfg, ids, dtype, qk_norm, False)


def last_attention(w, cfg, ids: Sequence[int], dtype=torch.float64, qk_norm: bool = True) -> torch.Tensor:
    """the last layer's attention probabilities of one sequence -> [heads, S, S]"""
    return _forward(w, cfg, ids, dtype, qk_norm, True)


def find_part(thread: Sequence[int], part: Sequence[int]) -> Tuple[int, int]:
    """(start, start + len(part) - 1) of the first occurrence of ``part`` in ``thread``; ValueError if it is absent"""
    thread, part = list(thread), list(part)
    for i in range(len(thread) - len(part) + 1):
        if thread[i:i + len(part)] == part:
            return i, i + len(part) - 1
    raise ValueError("Sublist not found")


def block_mean(A: np.ndarray, rows: Tuple[int, int], cols: Tuple[int, int]) -> float:
    a = A[:, rows[0]:rows[1], cols[0]:cols[1]]
    return float(a.mean()) if a.size else float("nan")


def attention_scores(A: np.ndarray, thread_ids: Sequence[int], query_ids: Sequence[int], answer_ids: Sequence[int],
                     context_ids: Sequence[Sequence[int]], include_query: bool = True) -> List[np.float64]:
    q, a = find_part(thread_ids, query_ids), find_part(thread_ids, answer_ids)
    docs = [find_part(thread_ids, c) for c in context_ids]
    total = [v for v in (block_mean(A, q, q), block_mean(A, q, a), block_mean(A, a, a), block_mean(A, a, q)) if v > 0]
    per_doc = []
    for d in docs:
        vals = [block_mean(A, a, d), block_mean(A, d, a)]
        if include_query:
            vals += [block_mean(A, q, d), block_mean(A, d, q)]
        kept = [v for v in vals if v > 0]
        total += kept
        per_doc.append(np.mean(kept) if kept else np.float64("nan"))
    mean_total = np.mean(total) if total else np.float64("nan")
    return [np.float64(s / mean_total) for s in per_doc]
