"""GPU: the kernels of one decode step that only whole-model generation reached before, one at a time against float64 or
bit for bit: Llama's q / k step (``qk_norm_rope_kernel<false>``: rotary without the per-head RMSNorm, llama3-scaled
tables, positions to 131 071), Qwen3's at one token, the KV-cache append (``rmu_debug_kv_append``), decode attention
with more than 8 query heads per kv head (grid z > 1), and the three chained at kernel level: q / k step, a prefill
append, a one-row append and decode attention against float64 causal attention of the last row."""
from __future__ import annotations

import functools
import math

import numpy as np
import pytest
import torch

from ragmeup_b200.weights import LlamaConfig, rope_table
from test_encoder_kernels_gpu import SENT16, U, _sentinel16, _split_err, _split_ok

pytestmark = pytest.mark.gpu
D = 128                                 # head_dim of every decoder the generation path runs
LOG2E = math.log2(math.e)
QS = LOG2E / math.sqrt(D)
# Llama's q / k step: out_c = (x_c cos - x_p sin) * sc in fp32, x_p the other half of the head.  Two products, the sum
# and the q-scale product round against at most (|x_c| |cos| + |x_p| |sin|) |sc|: c = 4 in units of u times that; the
# split adds 2^-22 |out|.
C_ROPE = 4.0
ATT_ABS = 2e-5                          # tests/test_generation_gpu.py's decode-attention bound


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def _split(x):
    hi = x.half()
    return hi, (x - hi.float()).half()


@functools.lru_cache(maxsize=None)
def _llama_tables():
    cfg = LlamaConfig()                 # Llama-3.1-8B: theta 500 000, llama3 scaling, 131 072 positions
    return tuple(torch.from_numpy(t).cuda() for t in rope_table(cfg.rope_theta, D, cfg.max_pos, cfg.rope_scaling))


def _qk_step(x, pos, heads, kv, tables, qn=None, kn=None, slack=0):
    """rmu_debug_qk_norm_rope on fp32 rows x [T, NH 128] -> (hi, lo, range flag), the planes with `slack` rows of NaN
    past T"""
    L = _lib()
    T = x.shape[0]
    hi = torch.full((T + slack, x.shape[1]), float("nan"), dtype=torch.float16, device="cuda")
    lo = torch.full_like(hi, float("nan"))
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(L.lib().rmu_debug_qk_norm_rope(_ptr(x), T, heads, kv, _ptr(pos), _ptr(qn), _ptr(kn), 1e-6, QS,
                                           _ptr(tables[0]), _ptr(tables[1]), tables[0].shape[0], _ptr(hi), _ptr(lo),
                                           _ptr(flag), L.stream_ptr()), "rmu_debug_qk_norm_rope")
    torch.cuda.synchronize()
    return hi, lo, int(flag.item())


def _rope64(y, pos, tables):
    """float64 rotate-half of y [T, n, 128] at the positions clamped into the tables; returns (rotated, the magnitude
    |y_c| |cos| + |y_p| |sin| its fp32 evaluation rounds against)"""
    p = pos.long().clamp(0, tables[0].shape[0] - 1)
    c, s = tables[0].double()[p][:, None, :], tables[1].double()[p][:, None, :]
    c, s = torch.cat([c, c], -1), torch.cat([s, s], -1)
    partner = torch.cat([y[..., D // 2:], y[..., :D // 2]], -1)
    sign = torch.cat([-torch.ones(D // 2), torch.ones(D // 2)]).to(y)
    return y * c + sign * partner * s, y.abs() * c.abs() + partner.abs() * s.abs()


# ------------------------------------------------------------------------------------------------- the q / k step
@pytest.mark.parametrize("heads,kv", [(32, 8), (8, 2), (4, 4)])
@pytest.mark.parametrize("T", [1, 700])
def test_llama_qk_step_matches_float64(cuda, heads, kv, T):
    """qk_norm_rope_kernel<false>: q and k rotated with Llama-3.1's llama3-scaled tables, q times log2(e) / sqrt(128),
    v copied; positions 0, 1, the table's last two, one below 0 and one past the table (both clamp)"""
    gen = torch.Generator(device="cuda").manual_seed(heads * 1000 + kv * 10 + T)
    tabs = _llama_tables()
    rows = tabs[0].shape[0]
    NH = heads + 2 * kv
    x = torch.randn((T, NH * D), device="cuda", generator=gen) * 3.0
    pos = torch.randint(0, rows, (T,), device="cuda", generator=gen, dtype=torch.int32)
    if T == 1:
        pos[0] = 123457
    else:
        pos[:6] = torch.tensor([0, 1, rows - 2, rows - 1, -5, rows + 9], dtype=torch.int32)
    hi, lo, flag = _qk_step(x, pos, heads, kv, tabs)
    _split_ok(hi, lo)
    assert flag == 0
    got = (hi.double() + lo.double()).view(T, NH, D)
    X = x.double().view(T, NH, D)
    want, mag = _rope64(X[:, :heads + kv], pos, tabs)
    sc = torch.ones(heads + kv, dtype=torch.float64, device="cuda")
    sc[:heads] = float(np.float32(QS))
    want, mag = want * sc[None, :, None], mag * sc[None, :, None]
    err = (got[:, :heads + kv] - want).abs() - _split_err(want)
    ratio = float((err.clamp(min=0) / (U * mag + 1e-300)).max())
    print(f"\nllama qk step heads={heads} kv={kv} T={T}: worst |err| / (u (|x||cos| + |x_p||sin|) sc) = {ratio:.3g}")
    assert ratio <= C_ROPE, f"q / k step error {ratio:.3g} exceeds {C_ROPE}"
    vh, vl = _split(x.view(T, NH, D)[:, heads + kv:])            # v: the split of x, bit for bit
    assert torch.equal(hi.view(T, NH, D)[:, heads + kv:].view(torch.int16), vh.view(torch.int16))
    assert torch.equal(lo.view(T, NH, D)[:, heads + kv:].view(torch.int16), vl.view(torch.int16))
    # an output past fp16's range (here a v element of the last row) sets the flag
    x2 = x.clone()
    x2[T - 1, -1] = 7e4
    assert _qk_step(x2, pos, heads, kv, tabs)[2] == 1


def test_qwen3_qk_step_one_token_far_position(cuda):
    """qk_norm_rope_kernel<true> at T = 1 and position 40 000 of Qwen3's 40 960-row table"""
    gen = torch.Generator(device="cuda").manual_seed(40000)
    heads, kv = 16, 8
    NH = heads + 2 * kv
    tabs = tuple(torch.from_numpy(t).cuda() for t in rope_table(1000000.0, D, 40960))
    x = torch.randn((1, NH * D), device="cuda", generator=gen) * 3.0
    qn = 1.0 + 0.2 * torch.randn(D, device="cuda", generator=gen)
    kn = 1.0 + 0.2 * torch.randn(D, device="cuda", generator=gen)
    pos = torch.tensor([40000], dtype=torch.int32, device="cuda")
    hi, lo, flag = _qk_step(x, pos, heads, kv, tabs, qn, kn)
    _split_ok(hi, lo)
    X = x.double().view(1, NH, D)

    def norm(v, w):
        return w.double() * (v * torch.rsqrt(v.pow(2).mean(-1, keepdim=True) + 1e-6))
    want = X.clone()
    want[:, :heads] = _rope64(norm(X[:, :heads], qn), pos, tabs)[0] * float(np.float32(QS))
    want[:, heads:heads + kv] = _rope64(norm(X[:, heads:heads + kv], kn), pos, tabs)[0]
    got = (hi.double() + lo.double()).view(1, NH, D)
    err = float(((got - want).abs() / want.abs().amax(-1, keepdim=True)).max())
    print(f"\nqwen3 qk step T=1 pos=40000: max |err| / head max = {err:.3g}")
    assert err <= 2e-6 and flag == 0                              # tests/test_qwen3_gpu.py's bound


# ------------------------------------------------------------------------------------------------- the KV-cache append
def _append(hi, lo, T, heads, kv, pos0, cap, cache):
    L = _lib()
    L.check(L.lib().rmu_debug_kv_append(_ptr(hi), _ptr(lo), T, heads, kv, pos0, cap, _ptr(cache), L.stream_ptr()),
            "rmu_debug_kv_append")
    torch.cuda.synchronize()


def _cache(kv, cap):
    """one layer's cache [4 (K hi, K lo, V hi, V lo), kv, cap, 128] of sentinels"""
    return _sentinel16(4 * kv * cap, D).view(4, kv, cap, D)


@pytest.mark.parametrize("heads,kv,T,pos0,cap", [
    (32, 8, 1, 49, 50),                # one decode token into the cache's last row
    (8, 2, 4097, 0, 4100),             # a prefill from position 0
    (4, 1, 7, 3, 16),                  # kv_heads 1
    (16, 2, 65, 100, 1000),
])
def test_kv_append_writes_exactly_its_rows(cuda, heads, kv, T, pos0, cap):
    """rows pos0 .. pos0 + T - 1 of K hi / K lo / V hi / V lo are the k and v head planes bit for bit; every other cache
    element keeps its sentinel"""
    gen = torch.Generator(device="cuda").manual_seed(heads + 7 * kv + T + pos0)
    NH = heads + 2 * kv
    hi, lo = _split(torch.randn((T + 2, NH * D), device="cuda", generator=gen))   # two rows of slack past T
    cache = _cache(kv, cap)
    _append(hi, lo, T, heads, kv, pos0, cap, cache)
    c = cache.view(torch.int16)
    ph, pl = hi[:T].view(T, NH, D).transpose(0, 1), lo[:T].view(T, NH, D).transpose(0, 1)   # [NH, T, 128]
    want = [ph[heads:heads + kv], pl[heads:heads + kv], ph[heads + kv:], pl[heads + kv:]]
    for i, name in enumerate(("K hi", "K lo", "V hi", "V lo")):
        assert torch.equal(c[i, :, pos0:pos0 + T], want[i].view(torch.int16)), f"{name} rows differ from the planes"
    keep = torch.ones(cap, dtype=torch.bool, device="cuda")
    keep[pos0:pos0 + T] = False
    assert (c[:, :, keep] == SENT16).all(), "the append wrote cache rows outside pos0 .. pos0 + T - 1"


# ------------------------------------------------------------------------------------------------- decode attention
def _decode(qh, ql, kv_planes, heads, kv, cap, n):
    """rmu_debug_attention_decode with a workspace of NaN (a partial never written shows in the output)"""
    L = _lib()
    ws = torch.full((heads * ((n + 63) // 64) * 130,), float("nan"), device="cuda")
    ch = torch.empty(heads * D, dtype=torch.float16, device="cuda")
    cl = torch.empty_like(ch)
    L.check(L.lib().rmu_debug_attention_decode(_ptr(qh), _ptr(ql), _ptr(kv_planes), heads, kv, cap, n, _ptr(ws),
                                               ws.numel(), _ptr(ch), _ptr(cl), L.stream_ptr()),
            "rmu_debug_attention_decode")
    torch.cuda.synchronize()
    return ch, cl


def _decode_ref(q, k, v, G):
    """float64 softmax attention of q [heads, 128] (log2 units) over k, v [kv, n, 128]; head h reads kv head h / G"""
    kr, vr = k.repeat_interleave(G, 0), v.repeat_interleave(G, 0)
    s = torch.einsum("hd,hjd->hj", q, kr) * math.log(2.0)
    return torch.einsum("hj,hjd->hd", s.softmax(-1), vr)


@pytest.mark.parametrize("G", [12, 16])
@pytest.mark.parametrize("n", [1, 64, 65, 4097])
def test_attention_decode_large_groups(cuda, G, n):
    """G = heads / kv_heads > 8 takes ceil(G / 8) CTAs per (kv head, split): G = 12 leaves a partial second group"""
    kv = 2
    heads, cap = G * kv, n + 5
    gen = torch.Generator(device="cuda").manual_seed(n * 31 + G)
    q = torch.randn(heads, D, device="cuda", generator=gen) * QS
    k = torch.randn(kv, cap, D, device="cuda", generator=gen) * 2.0
    v = torch.randn(kv, cap, D, device="cuda", generator=gen)
    qh, ql = _split(q)
    kh, kl = _split(k)
    vh, vl = _split(v)
    planes = torch.stack([kh, kl, vh, vl]).contiguous()
    outs = [_decode(qh, ql, planes, heads, kv, cap, n) for _ in range(2)]
    assert torch.equal(outs[0][0].view(torch.int16), outs[1][0].view(torch.int16)) and \
        torch.equal(outs[0][1].view(torch.int16), outs[1][1].view(torch.int16)), "repeated calls differ"
    _split_ok(*outs[0])
    got = (outs[0][0].double() + outs[0][1].double()).view(heads, D)
    want = _decode_ref(qh.double() + ql.double(), (kh.double() + kl.double())[:, :n], (vh.double() + vl.double())[:, :n], G)
    err = float((got - want).abs().max())
    print(f"\ndecode attention G={G} n={n}: max |err| = {err:.3g}")
    assert err < ATT_ABS, err


# ------------------------------------------------------------------------------------------------- one decode step's layout
@pytest.mark.parametrize("T", [63, 64, 1000])
def test_prefill_append_decode_chain_matches_causal_float64(cuda, T):
    """q / k step on T + 1 rows, the first T appended as a prefill, row T appended alone at pos0 = T, then decode
    attention of row T over n = T + 1 keys: float64 causal attention of the planes' last row.  A cache whose positions or
    heads do not line up with the planes fails here without a model."""
    heads, kv = 8, 2
    G, NH = heads // kv, heads + 2 * kv
    gen = torch.Generator(device="cuda").manual_seed(T)
    tabs = _llama_tables()
    x = torch.randn((T + 1, NH * D), device="cuda", generator=gen)
    pos = torch.arange(T + 1, dtype=torch.int32, device="cuda")
    hi, lo, flag = _qk_step(x, pos, heads, kv, tabs, slack=1)
    assert flag == 0
    cap = T + 5
    cache = _cache(kv, cap)
    _append(hi, lo, T, heads, kv, 0, cap, cache)
    _append(hi[T:], lo[T:], 1, heads, kv, T, cap, cache)
    ch, cl = _decode(hi[T, :heads * D], lo[T, :heads * D], cache, heads, kv, cap, T + 1)
    got = (ch.double() + cl.double()).view(heads, D)
    X = (hi[:T + 1].double() + lo[:T + 1].double()).view(T + 1, NH, D)
    want = _decode_ref(X[T, :heads], X[:, heads:heads + kv].transpose(0, 1), X[:, heads + kv:].transpose(0, 1), G)
    err = float((got - want).abs().max())
    print(f"\nq / k step -> append -> decode, T={T}: max |err| = {err:.3g}")
    assert err < ATT_ABS, err
    assert (cache.view(torch.int16)[:, :, T + 1:] == SENT16).all()
