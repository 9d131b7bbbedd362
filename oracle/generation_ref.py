"""Oracle for text generation on the GPU decoder (``rmu_decoder_generate``, ``llms.HuggingFacePipeline``).  TEST
INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

* ``logits``: ``lm_head . decoder_attention_ref.hidden(...)[-1]`` in float64.
* The four processors of transformers' sampling path, restated in float64: ``repetition_penalty`` (x < 0 ? x p : x / p
  on every id seen), ``temperature`` (x / t), ``top_k`` (every x >= the k-th largest survives, the rest -inf) and
  ``top_p`` (sorted ascending, the cumulative softmax <= 1 - p is removed, the last always kept).  torch.sort does
  not specify the order of equal values; here they go by descending id, so the lowest id is kept first, as the sampler
  keeps it.
* ``candidates`` / ``draw``: the GPU sampler's rule after the processors: at most 256 survivors (lowest ids among ties
  at the k-th value), largest first with the lowest id first among equal values, and the first whose cumulative
  weight exp(x - max) exceeds u times the kept total.
* ``philox_uniform``: the sampler's Philox4x32-10 uniform of (seed, step).
* ``generate``: greedy or sampled generation by full recomputation of every step.
PARITY STATUS: the processors and greedy generation are checked against transformers (LogitsProcessors,
LlamaForCausalLM / Qwen3ForCausalLM.generate in float64) in tests/test_generation_cpu.py.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch

from oracle import decoder_attention_ref as da

CAP = 256


def logits(w, lm_head, cfg, ids: Sequence[int], qk_norm: bool) -> np.ndarray:
    h = da.hidden(w, cfg, ids, torch.float64, qk_norm)[-1]
    return (torch.as_tensor(lm_head, dtype=torch.float64) @ h).numpy()


def repetition_penalty(x: np.ndarray, seen: Sequence[int], p: float) -> np.ndarray:
    x = np.array(x, dtype=np.float64)
    ids = np.unique(np.asarray(list(seen), dtype=np.int64))
    v = x[ids]
    x[ids] = np.where(v < 0, v * p, v / p)
    return x


def temperature(x: np.ndarray, t: float) -> np.ndarray:
    return np.asarray(x, dtype=np.float64) / t


def top_k(x: np.ndarray, k: int) -> np.ndarray:
    x = np.asarray(x, dtype=np.float64)
    k = min(k, x.size)
    kth = np.sort(x)[::-1][k - 1]
    return np.where(x < kth, -np.inf, x)


def top_p(x: np.ndarray, p: float) -> np.ndarray:
    x = np.asarray(x, dtype=np.float64)
    order = np.lexsort((-np.arange(x.size), x))          # value ascending, then id descending
    s = x[order]
    e = np.exp(s - s[-1])
    cum = np.cumsum(e / e.sum())
    remove = cum <= 1 - p
    remove[-1] = False
    out = x.copy()
    out[order[remove]] = -np.inf
    return out


def candidates(x: np.ndarray, k: int) -> np.ndarray:
    """the sampler's survivors of top-k (at most 256: the lowest ids among ties at the k-th value), largest first, the
    lowest id first among equal values"""
    x = np.asarray(x, dtype=np.float64)
    order = np.lexsort((np.arange(x.size), -x))          # value descending, then id ascending
    kth = x[order[min(k, x.size) - 1]]
    keep = [i for i in order if x[i] >= kth][:CAP]
    return np.asarray(keep, dtype=np.int64)


def kept(x: np.ndarray, cand: np.ndarray, p: float) -> np.ndarray:
    """top-p over the candidates (largest first): the prefix whose ascending cumulative softmax stays above 1 - p"""
    v = x[cand]
    w = np.exp(v - v[0])
    total = w.sum()
    n = len(cand)
    suf = 0.0
    for r in range(len(cand) - 1, 0, -1):
        suf += w[r]
        if suf / total <= 1 - p:
            n = r
        else:
            break
    return cand[:n]


def probabilities(x: np.ndarray, k: int, p: float) -> np.ndarray:
    """the sampler's distribution over ids after the processors (x already penalised and tempered)"""
    c = kept(x, candidates(x, k), p)
    w = np.exp(x[c] - x[c[0]])
    out = np.zeros(x.size)
    out[c] = w / w.sum()
    return out


def draw(x: np.ndarray, k: int, p: float, u: float) -> int:
    c = kept(x, candidates(x, k), p)
    w = np.exp(x[c] - x[c[0]])
    target, cum = u * w.sum(), 0.0
    for r, wr in enumerate(w):
        cum += wr
        if target < cum:
            return int(c[r])
    return int(c[-1])


def greedy(x: np.ndarray) -> int:
    x = np.asarray(x)
    return int(np.flatnonzero(x == x.max())[0])


def philox4x32_10(ctr: Sequence[int], key: Sequence[int]) -> List[int]:
    """Philox4x32-10 (Salmon et al., SC'11; Random123's philox4x32): four 32-bit counter words, two key words"""
    M = 0xFFFFFFFF
    c = [int(x) & M for x in ctr]
    k0, k1 = int(key[0]) & M, int(key[1]) & M
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k0) & M, p1 & M, ((p0 >> 32) ^ c[3] ^ k1) & M, p0 & M]
        k0, k1 = (k0 + 0x9E3779B9) & M, (k1 + 0xBB67AE85) & M
    return c


def philox_uniform(seed: int, step: int) -> float:
    """the sampler's uniform: counter (step, 0), key seed, the first output word's high 24 bits / 2^24"""
    M = 0xFFFFFFFF
    c = philox4x32_10([step & M, (step >> 32) & M, 0, 0], [seed & M, (seed >> 32) & M])
    return (c[0] >> 8) / 16777216.0


def generate(w, lm_head, cfg, ids: Sequence[int], max_new_tokens: int, qk_norm: bool, do_sample: bool = False,
             temp: float = 1.0, k: int = 50, p: float = 1.0, penalty: float = 1.0, eos: Sequence[int] = (),
             seed: int = 0) -> List[int]:
    seq, out = list(ids), []
    for step in range(max_new_tokens):
        x = repetition_penalty(logits(w, lm_head, cfg, seq, qk_norm), seq, penalty)
        if do_sample:
            t = draw(temperature(x, temp), k, p, philox_uniform(seed, step))
        else:
            t = greedy(x)
        out.append(t)
        seq.append(t)
        if t in eos or len(seq) >= cfg.max_pos:
            break
    return out
