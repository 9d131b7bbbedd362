"""Batched generation on the GPU decoder (rmu_decoder_generate_batch): each row of a batch is bit for bit what
rmu_decoder_generate returns for that prompt and seed, tokens and logits, on split and NF4 handles, greedy and sampled,
across shared prefixes that straddle the attention kernels' 16-row and 64-key boundaries; the multi-row NF4 GEMV
(rmu_debug_nf4_gemv_rows) row for row against the one-row GEMV; the batched kernels one at a time against their
one-sequence forms (decode attention with the prefix mapping, the cached-key prefill attention, the per-row sampler),
at 1, 2, 4, 5, 8 and 16 query heads per kv head; the refusals; and single calls around a batch."""
from __future__ import annotations

import ctypes as C
import gc
from dataclasses import replace

import numpy as np
import pytest
import torch

import make_golden_generate as mg
from oracle import generation_ref as gref
from oracle import nf4_ref as nf4

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release_torch_cache():
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    yield


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _split(x):
    hi = x.to(torch.float16)
    return hi, (x - hi.float()).to(torch.float16)


# ------------------------------------------------------------------------------------------------ multi-row GEMV
def _quantize(w16):
    L = _lib()
    n = w16.numel()
    codes = torch.empty(n // 2, dtype=torch.uint8, device="cuda")
    absmax = torch.empty(n // 64, dtype=torch.float32, device="cuda")
    L.check(L.lib().rmu_debug_nf4_quantize(w16.data_ptr(), n, codes.data_ptr(), absmax.data_ptr(), L.stream_ptr()),
            "quantize")
    return codes, absmax


def _gemv_call(fn, mode, M, x_hi, x_lo, codes, absmax, N, K, bias, res):
    L = _lib()
    if mode == 7:
        hi = torch.full((M, N // 2), float("nan"), dtype=torch.float16, device="cuda")
        lo = torch.full_like(hi, float("nan"))
        out = None
    else:
        out = res.clone() if res is not None else torch.full((M, N), float("nan"), device="cuda")
        hi = lo = None
    args = [x_hi.data_ptr(), x_lo.data_ptr(), codes.data_ptr(), absmax.data_ptr(), N, K, bias.data_ptr(),
            None if res is None else (out.data_ptr() if mode == 6 else res.data_ptr()),
            None if out is None else out.data_ptr(), None if hi is None else hi.data_ptr(),
            None if lo is None else lo.data_ptr(), None, L.stream_ptr()]
    if fn == "rows":
        L.check(L.lib().rmu_debug_nf4_gemv_rows(mode, M, *args), "gemv_rows")
    else:
        L.check(L.lib().rmu_debug_nf4_gemv(mode, *args), "gemv")
    torch.cuda.synchronize()
    return out if out is not None else torch.cat([hi, lo], 1)


@pytest.mark.parametrize("K", [4096, 14336])
@pytest.mark.parametrize("mode", [0, 6, 7])
def test_gemv_rows_equal_one_row_launches(mode, K):
    """every row of an M-row launch (M = 2 .. 16) equals the one-row GEMV on that row bit for bit, so each carries
    the one-row GEMV's float64 bound (test_nf4_gpu.test_gemv_modes_against_float64)"""
    N = 512
    g = torch.Generator(device="cuda").manual_seed(K + mode)
    w16 = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(torch.float16)
    codes, absmax = _quantize(w16)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    for M in (2, 3, 4, 5, 8, 9, 16):
        x = torch.randn(M, K, device="cuda", generator=g) * 2
        x_hi, x_lo = _split(x)
        res = torch.randn(M, N, device="cuda", generator=g) if mode == 6 else None
        got = _gemv_call("rows", mode, M, x_hi, x_lo, codes, absmax, N, K, bias, res)
        for m in range(M):
            one = _gemv_call("one", mode, 1, x_hi[m].contiguous(), x_lo[m].contiguous(), codes, absmax, N, K, bias,
                             None if res is None else res[m:m + 1].contiguous())
            assert torch.equal(got[m].view(torch.int32 if got.dtype == torch.float32 else torch.int16),
                               one[0].view(torch.int32 if one.dtype == torch.float32 else torch.int16)), (M, m)


def test_gemv_rows_refusals():
    L = _lib()
    z = torch.zeros(64, device="cuda")
    p = z.data_ptr()
    assert L.lib().rmu_debug_nf4_gemv_rows(0, 0, p, p, p, p, 128, 64, p, None, p, None, None, None, None) == -1
    assert L.lib().rmu_debug_nf4_gemv_rows(0, 17, p, p, p, p, 128, 64, p, None, p, None, None, None, None) == -1
    assert L.lib().rmu_debug_nf4_gemv_rows(3, 2, p, p, p, p, 128, 64, p, None, p, None, None, None, None) == -1
    assert L.lib().rmu_debug_nf4_gemv_rows(0, 2, p, p, p, p, 100, 64, p, None, p, None, None, None, None) == -3


# ------------------------------------------------------------------------------------------------ whole calls
def _handle(kind, weights="split", max_pos=8192, cfg_w_lm=None):
    from ragmeup_b200.encoder import BertEncoder
    cfg, w, lm = cfg_w_lm or mg.model(kind, max_pos=max_pos)
    enc = BertEncoder(cfg, w, with_head=False)
    L = _lib()
    if weights == "nf4":
        enc._check(L.lib().rmu_decoder_quantize_nf4(enc._h, L.stream_ptr()), "rmu_decoder_quantize_nf4")
    enc._check(L.lib().rmu_decoder_set_lm_head(enc._h, np.ascontiguousarray(lm).ctypes.data), "set_lm_head")
    return cfg, w, lm, enc


def _sampling(do_sample=False, temp=1.0, k=50, p=1.0, penalty=1.0, eos=()):
    L = _lib()
    return L.SamplingC(int(do_sample), temp, p, penalty, k, len(eos), (C.c_int32 * L.MAX_EOS)(*eos))


def _single(enc, V, ids, s, seed, max_new):
    L = _lib()
    prompt = np.ascontiguousarray(ids, dtype=np.int32)
    out = np.zeros(max_new, dtype=np.int32)
    logits = np.full((max_new, V), np.nan, dtype=np.float32)
    n = C.c_int32(0)
    rc = L.lib().rmu_decoder_generate(enc._h, prompt.ctypes.data, len(prompt), C.byref(s), seed, max_new,
                                      out.ctypes.data, C.byref(n), logits.ctypes.data, L.stream_ptr())
    assert rc == 0, L.lib().rmu_last_error()
    return out[:n.value].tolist(), logits[:n.value]


def _batch(enc, V, prompts, s, seeds, max_new):
    L = _lib()
    B = len(prompts)
    ids = np.ascontiguousarray([t for p in prompts for t in p], dtype=np.int32)
    cu = np.ascontiguousarray(np.cumsum([0] + [len(p) for p in prompts]), dtype=np.int32)
    sd = np.ascontiguousarray(seeds, dtype=np.uint64)
    out = np.full((B, max_new), -7, dtype=np.int32)
    n = np.zeros(B, dtype=np.int32)
    logits = np.full((B, max_new, V), np.nan, dtype=np.float32)
    rc = L.lib().rmu_decoder_generate_batch(enc._h, ids.ctypes.data, cu.ctypes.data, B, C.byref(s), sd.ctypes.data,
                                            max_new, out.ctypes.data, n.ctypes.data, logits.ctypes.data, L.stream_ptr())
    return rc, out, n, logits


def _prompts(V, B, P, seed, lens=None):
    """B prompts sharing their first P tokens (then distinct first own tokens), own lengths `lens` or 1 .. 37"""
    rng = np.random.default_rng(seed)
    prefix = rng.integers(0, V, P).tolist()
    lens = lens or [1 + (7 * b + seed) % 37 for b in range(B)]
    out = []
    for b in range(B):
        own = rng.integers(0, V, lens[b]).tolist()
        own[0] = (b * 13 + 5) % V
        out.append(prefix + own)
    return out


def _check_parity(enc, V, prompts, s, seeds, max_new):
    rc, out, n, logits = _batch(enc, V, prompts, s, seeds, max_new)
    assert rc == 0, _lib().lib().rmu_last_error()
    for b, p in enumerate(prompts):
        toks, lg = _single(enc, V, p, s, seeds[b], max_new)
        assert out[b, :n[b]].tolist() == toks, b
        assert np.array_equal(logits[b, :n[b]].view(np.int32), lg.view(np.int32)), b
        assert (out[b, n[b]:] == -7).all() and np.isnan(logits[b, n[b]:]).all()      # slots after the stop untouched
    return out, n


CASES = [  # (B, P, own lengths or None)
    (1, 0, [9]),
    (2, 0, None),
    (5, 1, None),
    (5, 63, [1, 2, 17, 40, 64]),
    (5, 64, None),
    (16, 64, None),
    (4, 300, [1, 30, 5, 90]),
]


@pytest.mark.parametrize("weights", ["split", "nf4"])
@pytest.mark.parametrize("kind", mg.KINDS)
def test_batch_equals_sequential(kind, weights):
    cfg, w, lm, enc = _handle(kind, weights)
    V = cfg.vocab_size
    for i, (B, P, lens) in enumerate(CASES):
        prompts = _prompts(V, B, P, 11 * i + 1, lens)
        seeds = [1000 + 17 * b for b in range(B)]
        _check_parity(enc, V, prompts, _sampling(penalty=1.2), seeds, 6)
        _check_parity(enc, V, prompts, _sampling(True, 0.8, 40, 0.9, 1.3), seeds, 6)
    # identical prompts (the prefix is capped to leave each one token), one-token prompts, eos stopping rows apart
    same = [_prompts(V, 1, 0, 3, [20])[0]] * 3
    _check_parity(enc, V, same, _sampling(True, 1.0, 50, 1.0), [1, 2, 3], 5)
    short = [[7], [9], [7, 8, 9, 10]]
    _check_parity(enc, V, short, _sampling(), [0, 0, 0], 5)
    prompts = _prompts(V, 6, 40, 5)
    out, _ = _check_parity(enc, V, prompts, _sampling(), [0] * 6, 8)
    eos = (int(out[0, 1]), int(out[3, 4]))
    _, n = _check_parity(enc, V, prompts, _sampling(eos=eos), [0] * 6, 8)
    assert len(set(n.tolist())) > 1                              # the rows stopped at different steps


def test_batch_stops_at_max_pos_and_alternates_with_single_calls():
    """rows stop at max_pos = 64 at different steps; a single call before and after a batch gives the same result, so
    the batch leaves the handle's KV cache usable for the single path"""
    cfg, w, lm, enc = _handle("llama", max_pos=64)
    V = cfg.vocab_size
    single_before = _single(enc, V, list(range(3, 33)), _sampling(), 0, 12)
    prompts = _prompts(V, 4, 20, 9, [40, 30, 2, 38])             # totals 60, 50, 22, 58
    _, n = _check_parity(enc, V, prompts, _sampling(), [0] * 4, 12)
    assert n.tolist() == [4, 12, 12, 6]
    single_after = _single(enc, V, list(range(3, 33)), _sampling(), 0, 12)
    assert single_before[0] == single_after[0]
    assert np.array_equal(single_before[1].view(np.int32), single_after[1].view(np.int32))


def test_batch_agrees_with_the_float64_oracle():
    cfg, w, lm, enc = _handle("qwen3")
    prompts = _prompts(cfg.vocab_size, 3, 24, 2, [3, 8, 1])
    rc, out, n, _ = _batch(enc, cfg.vocab_size, prompts, _sampling(penalty=1.2), [0, 0, 0], 6)
    assert rc == 0
    for b, p in enumerate(prompts):
        assert out[b, :n[b]].tolist() == gref.generate(w, lm, cfg, p, 6, qk_norm=True, penalty=1.2)


def test_batch_refusals():
    cfg, w, lm, enc = _handle("llama", max_pos=64)
    V = cfg.vocab_size
    L = _lib()
    ok = [[1, 2, 3], [1, 2, 4]]
    assert _batch(enc, V, ok, _sampling(), [0, 0], 3)[0] == 0
    assert _batch(enc, V, [[1]] * 17, _sampling(), [0] * 17, 3)[0] == -1                 # above the cap
    assert _batch(enc, V, [[1, 2], []], _sampling(), [0, 0], 3)[0] == -1                 # an empty prompt
    assert _batch(enc, V, [[1, 2], [V]], _sampling(), [0, 0], 3)[0] == -1                # an id out of range
    assert _batch(enc, V, [[1, 2], list(range(64))], _sampling(), [0, 0], 3)[0] == -1    # T >= max_pos
    assert _batch(enc, V, ok, _sampling(True, 1.0, 0), [0, 0], 3)[0] == -3               # top_k 0 when sampling
    assert _batch(enc, V, ok, _sampling(True, 0.0, 5), [0, 0], 3)[0] == -1
    assert _batch(enc, V, ok, _sampling(), [0, 0], 0)[0] == -1                           # max_new_tokens < 1
    ids = np.zeros(3, dtype=np.int32)
    cu = np.array([0, 3], dtype=np.int32)
    out = np.zeros(3, dtype=np.int32)
    n = np.zeros(1, dtype=np.int32)
    s = _sampling()
    assert L.lib().rmu_decoder_generate_batch(enc._h, ids.ctypes.data, cu.ctypes.data, 0, C.byref(s), ids.ctypes.data,
                                              3, out.ctypes.data, n.ctypes.data, None, None) == -1
    assert L.lib().rmu_decoder_generate_batch(enc._h, ids.ctypes.data, cu.ctypes.data, 1, C.byref(s), None, 3,
                                              out.ctypes.data, n.ctypes.data, None, None) == -1
    from ragmeup_b200.encoder import BertEncoder
    c2, w2, _ = mg.model("llama", max_pos=64)
    bare = BertEncoder(c2, w2, with_head=False)                  # no LM head
    assert L.lib().rmu_decoder_generate_batch(bare._h, ids.ctypes.data, cu.ctypes.data, 1, C.byref(s), ids.ctypes.data,
                                              3, out.ctypes.data, n.ctypes.data, None, None) == -1
    assert "LM head" in L.lib().rmu_last_error().decode()


def test_batch_range_error_returns_nothing():
    cfg_w_lm = mg.model("llama", scale=3000.0)
    cfg, w, lm, enc = _handle("llama", cfg_w_lm=cfg_w_lm)
    rc, out, n, _ = _batch(enc, cfg.vocab_size, [list(range(1, 30)), list(range(1, 20))], _sampling(), [0, 0], 3)
    assert rc == -4 and n.tolist() == [0, 0]


def test_llama_8b_shape_two_layers_nf4():
    """two layers of the Llama-3.1-8B shape on NF4, B = 8 prompts sharing 1 500 tokens: batch equals sequential"""
    from ragmeup_b200.weights import DECODER_PRESETS, synthetic_llama_weights
    cfg = replace(DECODER_PRESETS["llama-3.1-8b"], layers=2, vocab_size=2048, max_pos=4096)
    w = synthetic_llama_weights(cfg, seed=4)
    lm = (np.random.default_rng(4).standard_normal((cfg.vocab_size, cfg.hidden)) * 0.05).astype(np.float32)
    cfg, w, lm, enc = _handle("llama", "nf4", cfg_w_lm=(cfg, w, lm))
    del w
    prompts = _prompts(cfg.vocab_size, 8, 1500, 6, [200, 150, 1, 64, 65, 120, 30, 199])
    _check_parity(enc, cfg.vocab_size, prompts, _sampling(True, 0.6, 50, 0.9), list(range(8)), 4)


# ------------------------------------------------------------------------------------------------ kernels one at a time
@pytest.mark.parametrize("G", [1, 2, 4, 5, 8])
@pytest.mark.parametrize("P", [1, 63, 64, 65, 1000])
def test_decode_rows_prefix_mapping_equals_one_row_on_the_concatenated_cache(P, G):
    """rmu_debug_attention_decode_rows on rows of different own lengths (their 64-key splits straddle P) equals
    rmu_debug_attention_decode of each row on a cache holding [prefix | the row's own keys], bit for bit"""
    L = _lib()
    kv_heads = 2 if G < 8 else 1
    heads, own = G * kv_heads, [1, 70, 130]
    B, R = len(own), max(own)
    cap = P + B * R
    g = torch.Generator(device="cuda").manual_seed(P * 7 + G)
    q = torch.randn(B, heads * 128, device="cuda", generator=g) * (1.4426950408889634 / 128 ** 0.5)
    k = torch.randn(kv_heads, cap, 128, device="cuda", generator=g) * 2.0
    v = torch.randn(kv_heads, cap, 128, device="cuda", generator=g)
    qh, ql = _split(q)
    kh, kl = _split(k)
    vh, vl = _split(v)
    kv = torch.stack([kh, kl, vh, vl]).contiguous()
    pos = np.array([P + o - 1 for o in own], dtype=np.int32)
    shift = np.array([b * R for b in range(B)], dtype=np.int32)
    n = int(pos.max()) + 1
    ws = torch.empty(B * heads * ((n + 63) // 64) * 130 + 2 * B, device="cuda")
    ch = torch.empty(B, heads * 128, dtype=torch.float16, device="cuda")
    cl = torch.empty_like(ch)
    L.check(L.lib().rmu_debug_attention_decode_rows(qh.data_ptr(), ql.data_ptr(), heads * 128, B, kv.data_ptr(), heads,
                                                    kv_heads, cap, P, pos.ctypes.data, shift.ctypes.data, ws.data_ptr(),
                                                    ws.numel(), ch.data_ptr(), cl.data_ptr(), L.stream_ptr()),
            "decode_rows")
    torch.cuda.synchronize()
    for b in range(B):
        rows = torch.cat([torch.arange(P), torch.arange(P + b * R, P + b * R + own[b])]).cuda()
        cat = kv[:, :, rows].contiguous()
        nb = P + own[b]
        w1 = torch.empty(heads * ((nb + 63) // 64) * 130, device="cuda")
        oh = torch.empty(heads * 128, dtype=torch.float16, device="cuda")
        ol = torch.empty_like(oh)
        L.check(L.lib().rmu_debug_attention_decode(qh[b].contiguous().data_ptr(), ql[b].contiguous().data_ptr(),
                                                   cat.data_ptr(), heads, kv_heads, nb, nb, w1.data_ptr(), w1.numel(),
                                                   oh.data_ptr(), ol.data_ptr(), L.stream_ptr()), "decode")
        torch.cuda.synchronize()
        assert torch.equal(ch[b], oh) and torch.equal(cl[b], ol), b


@pytest.mark.parametrize("G", [1, 2, 5, 8, 16])
@pytest.mark.parametrize("P", [0, 1, 63, 64, 65, 1000])
def test_cached_prefill_attention_equals_the_full_causal_launch(P, G):
    """rmu_debug_attention_cached on the own rows of three sequences sharing P prefix rows (keys from the cache) equals
    rmu_debug_attention_causal's own rows on the full sequences, bit for bit: G = 1 runs 128-row CTAs (hpc 1), G = 5
    five query heads of 16 rows, G = 8 and 16 16-row CTAs of eight heads"""
    L = _lib()
    kv_heads = 2 if G <= 2 else 1
    heads, own = G * kv_heads, [1, 37, 130]
    NH = heads + 2 * kv_heads
    B, R = len(own), max(own)
    cap = P + B * R
    g = torch.Generator(device="cuda").manual_seed(P * 13 + G)

    def planes(rows):
        x = torch.randn(rows, NH, 128, device="cuda", generator=g)
        x[:, :heads] *= 1.4426950408889634 / 128 ** 0.5
        return _split(x.reshape(rows, NH * 128))

    pre = planes(P)
    suf = [planes(o) for o in own]
    full_hi = torch.cat([t for s in suf for t in (pre[0], s[0])])
    full_lo = torch.cat([t for s in suf for t in (pre[1], s[1])])
    cu_full = torch.tensor(np.cumsum([0] + [P + o for o in own]), dtype=torch.int32, device="cuda")
    fh = torch.empty(full_hi.shape[0], heads * 128, dtype=torch.float16, device="cuda")
    fl = torch.empty_like(fh)
    L.check(L.lib().rmu_debug_attention_causal(full_hi.data_ptr(), full_lo.data_ptr(), cu_full.data_ptr(), B, heads,
                                               kv_heads, P + R, fh.data_ptr(), fl.data_ptr(), L.stream_ptr()), "causal")
    # the cache: prefix rows 0 .. P - 1, sequence b's own key P + t at row P + t + b R
    kv = torch.zeros(4, kv_heads, cap, 128, dtype=torch.float16, device="cuda")

    def put(hi, lo, rows):
        h = hi.view(-1, NH, 128)
        lw = lo.view(-1, NH, 128)
        kv[0][:, rows] = h[:, heads:heads + kv_heads].transpose(0, 1)
        kv[1][:, rows] = lw[:, heads:heads + kv_heads].transpose(0, 1)
        kv[2][:, rows] = h[:, heads + kv_heads:].transpose(0, 1)
        kv[3][:, rows] = lw[:, heads + kv_heads:].transpose(0, 1)

    if P:
        put(pre[0], pre[1], torch.arange(P, device="cuda"))
    for b, s in enumerate(suf):
        put(s[0], s[1], torch.arange(P + b * R, P + b * R + own[b], device="cuda"))
    own_hi = torch.cat([s[0] for s in suf])
    own_lo = torch.cat([s[1] for s in suf])
    cu = torch.tensor(np.cumsum([0] + own), dtype=torch.int32, device="cuda")
    shift = torch.tensor([b * R for b in range(B) for _ in range(own[b])], dtype=torch.int32, device="cuda")
    ch = torch.full((own_hi.shape[0], heads * 128), float("nan"), dtype=torch.float16, device="cuda")
    cl = torch.full_like(ch, float("nan"))
    L.check(L.lib().rmu_debug_attention_cached(own_hi.data_ptr(), own_lo.data_ptr(), cu.data_ptr(), B, heads, kv_heads,
                                               kv.data_ptr(), cap, P, shift.data_ptr(), R, ch.data_ptr(), cl.data_ptr(),
                                               L.stream_ptr()), "cached")
    torch.cuda.synchronize()
    t0 = 0
    for b, o in enumerate(own):
        rows = slice(int(cu_full[b]) + P, int(cu_full[b]) + P + o)
        assert torch.equal(ch[t0:t0 + o], fh[rows]) and torch.equal(cl[t0:t0 + o], fl[rows]), b
        t0 += o


@pytest.mark.parametrize("sampled", [False, True])
def test_sampler_rows_equal_one_row_launches(sampled):
    """rmu_debug_sample_rows: row r (sequence seq[r]'s presence bits and seed, Philox at step 7) equals rmu_debug_sample
    on that row with u = philox(seed, 7): token, processed logits and presence bits"""
    L = _lib()
    V, B, nseq, step = 5000, 4, 6, 7
    words = (V + 31) // 32
    g = torch.Generator(device="cuda").manual_seed(int(sampled))
    logits = torch.randn(B, V, device="cuda", generator=g) * 3
    presence = torch.randint(0, 2 ** 31 - 1, (nseq, words), dtype=torch.int32, device="cuda", generator=g)
    presence &= torch.randint(0, 2 ** 31 - 1, (nseq, words), dtype=torch.int32, device="cuda", generator=g)
    seq = torch.tensor([3, 0, 5, 1], dtype=torch.int32, device="cuda")
    seeds_h = [91, 2 ** 63 + 5, 17, 3, 12345, 2 ** 40]
    seeds = torch.tensor(np.array(seeds_h, dtype=np.uint64).view(np.int64), device="cuda")
    s = _sampling(True, 0.7, 40, 0.9, 1.3) if sampled else _sampling(penalty=1.3)
    lg, pr = logits.clone(), presence.clone()
    tok = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    L.check(L.lib().rmu_debug_sample_rows(lg.data_ptr(), V, B, pr.data_ptr(), seq.data_ptr(), seeds.data_ptr(), step,
                                          C.byref(s), tok.data_ptr(), L.stream_ptr()), "sample_rows")
    torch.cuda.synchronize()
    for r in range(B):
        q = int(seq[r])
        l1, p1 = logits[r].clone(), presence[q].clone()
        t1 = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        u = gref.philox_uniform(seeds_h[q], step)
        L.check(L.lib().rmu_debug_sample(l1.data_ptr(), V, p1.data_ptr(), C.byref(s), float(u), t1.data_ptr(),
                                         L.stream_ptr()), "sample")
        torch.cuda.synchronize()
        assert int(tok[r]) == int(t1[0]), r
        assert torch.equal(lg[r].view(torch.int32), l1.view(torch.int32)) and torch.equal(pr[q], p1), r
    untouched = [q for q in range(nseq) if q not in seq.tolist()]
    assert torch.equal(pr[untouched], presence[untouched])


@pytest.mark.parametrize("G,kv_heads", [(1, 2), (5, 1), (8, 1)])
def test_batch_equals_sequential_across_group_sizes(G, kv_heads):
    """whole calls on Llama decoders with 1, 5 and 8 query heads per kv head (the prefill's 128-, 16- and 16-row
    causal CTAs), split and NF4, prefixes of 65 and 300 tokens"""
    from ragmeup_b200.weights import DECODER_PRESETS, synthetic_llama_weights
    cfg = replace(DECODER_PRESETS["tiny-llama"], vocab_size=1024, heads=G * kv_heads, kv_heads=kv_heads)
    w = synthetic_llama_weights(cfg, seed=G, scale=6.0)
    lm = (np.random.default_rng(G).standard_normal((cfg.vocab_size, cfg.hidden)) * 0.5).astype(np.float32)
    for weights in ("split", "nf4"):
        _, _, _, enc = _handle("llama", weights, cfg_w_lm=(cfg, w, lm))
        for P in (65, 300):
            prompts = _prompts(cfg.vocab_size, 4, P, P + G, [1, 20, 40, 130])
            _check_parity(enc, cfg.vocab_size, prompts, _sampling(penalty=1.2), [0] * 4, 5)
            _check_parity(enc, cfg.vocab_size, prompts, _sampling(True, 0.8, 40, 0.9, 1.2), [5, 6, 7, 8], 5)
        del enc
