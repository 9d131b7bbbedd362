"""NF4 decoder weights on the GPU: the quantiser and dequantiser bit for bit against oracle/nf4_ref.py, the decode GEMV's
three epilogues against float64 over the dequantised weights, and whole NF4 handles (rmu_decoder_quantize_nf4)
against the float64 forward on the oracle's dequantised weights, their memory, refusals and sharing."""
from __future__ import annotations

import ctypes as C
import gc

import numpy as np
import pytest
import torch

import make_golden_generate as mg
from oracle import decoder_attention_ref as da
from oracle import generation_ref as gref
from oracle import nf4_ref as nf4

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
PROJ = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj", "mlp.up_proj",
        "mlp.down_proj")
# (N, K) of the fused / blocked weights the handle holds: Llama-3.1-8B q | k | v, o, gate | up, down; Qwen3-0.6B's
LLAMA_8B = [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)]
QWEN3_06B = [(4096, 1024), (1024, 2048), (6144, 1024), (1024, 3072)]


@pytest.fixture(autouse=True)
def _release_torch_cache():
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    yield


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _rc(rc, what):
    L = _lib()
    assert rc == 0, (what, rc, L.lib().rmu_last_error())


def _quantize(w16: torch.Tensor):
    n = w16.numel()
    codes = torch.empty(n // 2, dtype=torch.uint8, device="cuda")
    absmax = torch.empty(n // 64, dtype=torch.float32, device="cuda")
    _rc(_lib().lib().rmu_debug_nf4_quantize(w16.data_ptr(), n, codes.data_ptr(), absmax.data_ptr(), _lib().stream_ptr()),
        "quantize")
    return codes, absmax


def _dequantize(codes, absmax):
    n = codes.numel() * 2
    hi = torch.empty(n, dtype=torch.float16, device="cuda")
    _rc(_lib().lib().rmu_debug_nf4_dequantize(codes.data_ptr(), absmax.data_ptr(), n, hi.data_ptr(), _lib().stream_ptr()),
        "dequantize")
    return hi


def _weights(N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = torch.randn(N, K, device="cuda", generator=g) * torch.exp(torch.randn(N, 1, device="cuda", generator=g))
    return (w * 0.05).to(torch.float16)


def _oracle_check(w16: torch.Tensor):
    codes, absmax = _quantize(w16)
    want_c, want_a = nf4.quantize(w16.cpu().numpy())
    assert np.array_equal(codes.cpu().numpy(), want_c.reshape(-1))
    assert np.array_equal(absmax.cpu().numpy().view(np.uint32), want_a.reshape(-1).view(np.uint32))
    hi = _dequantize(codes, absmax)
    assert np.array_equal(hi.cpu().numpy().view(np.uint16), nf4.dequantize(want_c, want_a).reshape(-1).view(np.uint16))


@pytest.mark.parametrize("N,K", [(256, 4096), (128, 14336), (512, 1024), (64, 3072)])
def test_quantiser_and_dequantiser_match_the_oracle(N, K):
    _oracle_check(_weights(N, K, N + K).reshape(N, K))


def test_quantiser_on_zero_spike_and_subnormal_blocks():
    w = _weights(64, 1024, 7).float()
    w[0] = 0                                                # all-zero blocks
    w[1] = 0
    w[1, 5::64] = -2.5                                      # one spike per block
    w[2] = torch.linspace(-6e-5, 6e-5, 1024, device="cuda")  # fp16 subnormals and their neighbours
    w[3] = torch.arange(1024, device="cuda").float() * 6e-8
    w[4, :64] = 65504.0
    _oracle_check(w.to(torch.float16))


def _gemv(mode, x_hi, x_lo, codes, absmax, N, K, bias, res=None, flag=None):
    L = _lib()
    if mode == 7:
        hi = torch.full((N // 2,), float("nan"), dtype=torch.float16, device="cuda")
        lo = torch.full((N // 2,), float("nan"), dtype=torch.float16, device="cuda")
        out = None
    else:
        out = res if res is not None else torch.full((N,), float("nan"), device="cuda")
        hi = lo = None
    _rc(L.lib().rmu_debug_nf4_gemv(mode, x_hi.data_ptr(), x_lo.data_ptr(), codes.data_ptr(), absmax.data_ptr(), N, K,
                                   bias.data_ptr(), None if res is None else res.data_ptr(),
                                   None if out is None else out.data_ptr(), None if hi is None else hi.data_ptr(),
                                   None if lo is None else lo.data_ptr(), None if flag is None else flag.data_ptr(),
                                   L.stream_ptr()), "gemv")
    torch.cuda.synchronize()
    return out.clone() if out is not None else (hi.double() + lo.double())


def _split(x):
    hi = x.to(torch.float16)
    return hi, (x - hi.float()).to(torch.float16)


@pytest.mark.parametrize("N,K", LLAMA_8B + QWEN3_06B)
def test_gemv_modes_against_float64(N, K):
    w16 = _weights(N, K, 3 * N + K)
    codes, absmax = _quantize(w16)
    W = _dequantize(codes, absmax).reshape(N, K).double()
    g = torch.Generator(device="cuda").manual_seed(K)
    x = torch.randn(K, device="cuda", generator=g) * 2
    x_hi, x_lo = _split(x)
    xd = x_hi.double() + x_lo.double()
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    acc = W @ xd
    mag = W.abs() @ xd.abs()
    err_acc = (K + 2) * U * mag                              # fp32 products and sums in a fixed order, x = fp32(hi + lo)
    # mode 0
    got = _gemv(0, x_hi, x_lo, codes, absmax, N, K, bias).double()
    want = acc + bias.double()
    assert ((got - want).abs() <= err_acc + 2 * U * want.abs() + 1e-30).all()
    assert torch.equal(_gemv(0, x_hi, x_lo, codes, absmax, N, K, bias).double(), got)     # the same bits on a repeat
    # mode 6, in place
    res0 = torch.randn(N, device="cuda", generator=g)
    res = res0.clone()
    got = _gemv(6, x_hi, x_lo, codes, absmax, N, K, bias, res=res).double()
    want = acc + bias.double() + res0.double()
    assert ((got - want).abs() <= err_acc + 4 * U * (acc.abs() + bias.double().abs() + res0.double().abs())).all()
    res = res0.clone()
    assert torch.equal(_gemv(6, x_hi, x_lo, codes, absmax, N, K, bias, res=res).double(), got)
    # mode 7: rows 128 b + i (gate) and 128 b + 64 + i (up) -> column 64 b + i
    idx = torch.arange(N // 2, device="cuda")
    gate_r = 128 * (idx // 64) + idx % 64
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    got = _gemv(7, x_hi, x_lo, codes, absmax, N, K, bias, flag=flag)
    gt, up = (acc + bias.double())[gate_r], (acc + bias.double())[gate_r + 64]
    want = torch.nn.functional.silu(gt) * up
    eg, eu = (err_acc + 2 * U * acc.abs())[gate_r], (err_acc + 2 * U * acc.abs())[gate_r + 64]
    bound = 1.1 * eg * up.abs() + torch.nn.functional.silu(gt).abs() * eu + 16 * U * want.abs() + 1e-30
    assert ((got - want).abs() <= bound).all(), float(((got - want).abs() / bound).max())
    assert int(flag.item()) == 0
    assert torch.equal(_gemv(7, x_hi, x_lo, codes, absmax, N, K, bias, flag=flag), got)
    # an output past 65504 sets the flag
    big = bias.clone()
    big[gate_r[5]] = 3e3
    big[gate_r[5] + 64] = 3e3
    _gemv(7, x_hi, x_lo, codes, absmax, N, K, big, flag=flag)
    assert int(flag.item()) == 1


def test_gemv_on_every_device():
    """the GEMV's shared-memory limit is a per-device attribute: a K = 14 336 row (56 KB of staged x, past the 48 KB
    default) runs on each GPU of the process, after one has already run it"""
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    N, K = 256, 14336
    outs = []
    for dev in range(torch.cuda.device_count()):
        with torch.cuda.device(dev):
            codes, absmax = _quantize(_weights(N, K, 5))
            x_hi, x_lo = _split(torch.linspace(-1, 1, K, device="cuda"))
            outs.append(_gemv(0, x_hi, x_lo, codes, absmax, N, K, torch.zeros(N, device="cuda")).cpu())
    assert all(torch.equal(o, outs[0]) for o in outs)


# ---------------------------------------------------------------------------------------------- whole NF4 handles
def _nf4_weights(w):
    return {k: (nf4.nf4_weight(v) if any(k.endswith(p + ".weight") for p in PROJ) else v) for k, v in w.items()}


def _convert(enc):
    _rc(_lib().lib().rmu_decoder_quantize_nf4(enc._h, _lib().stream_ptr()), "rmu_decoder_quantize_nf4")


def _generate(enc, ids, s, seed, max_new, logits=None):
    L = _lib()
    prompt = np.ascontiguousarray(ids, dtype=np.int32)
    out = np.zeros(max_new, dtype=np.int32)
    n = C.c_int32(0)
    rc = L.lib().rmu_decoder_generate(enc._h, prompt.ctypes.data, len(prompt), C.byref(s), seed, max_new,
                                      out.ctypes.data, C.byref(n), None if logits is None else logits.ctypes.data,
                                      L.stream_ptr())
    return rc, out[:n.value].tolist()


def _sampling(do_sample=False, temp=1.0, k=50, p=1.0, penalty=1.0):
    L = _lib()
    return L.SamplingC(int(do_sample), temp, p, penalty, k, 0, (C.c_int32 * L.MAX_EOS)())


def _handle_bytes(cfg):
    H, F, QD, KD = cfg.hidden, cfg.ffn, cfg.heads * 128, cfg.kv_heads * 128
    shapes = [(QD + 2 * KD, H), (H, QD), (2 * F, H), (H, F)]
    n = sum(a * b for a, b in shapes)
    return cfg.layers * (n // 2 + n // 64 * 4 - 4 * n) + 4 * max(a * b for a, b in shapes)


def test_conversion_frees_what_it_states():
    """a handle whose planes are each larger than the driver's 2 MB pages: the device memory the driver reports free
    grows by the conversion's stated saving (split planes freed, codes, absmax and the scratch allocated), to the
    driver's granularity of up to 2 MB per allocation made or freed"""
    from dataclasses import replace
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import DECODER_PRESETS, synthetic_llama_weights
    cfg = replace(DECODER_PRESETS["tiny-llama"], hidden=2048, ffn=8192, heads=16, kv_heads=4, layers=3,
                  vocab_size=1024, max_pos=4096)
    enc = BertEncoder(cfg, synthetic_llama_weights(cfg, seed=2), with_head=False)
    L = _lib()
    _dequantize(*_quantize(torch.zeros(64, dtype=torch.float16, device="cuda")))   # loads the NF4 kernels' module
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    _convert(enc)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    peak, delta = C.c_int64(), C.c_int64()
    _rc(L.lib().rmu_debug_nf4_conversion(enc._h, C.byref(peak), C.byref(delta)), "conversion")
    assert peak.value <= 0 and delta.value == _handle_bytes(cfg)
    allocations = cfg.layers * 4 * 4 + 2
    assert abs((free1 - free0) + delta.value) <= allocations * (2 << 20), (free1 - free0, delta.value)
    assert -delta.value > 4 * allocations * (2 << 20)                    # the saving dwarfs the granularity


@pytest.mark.parametrize("kind", mg.KINDS)
def test_nf4_handle_against_float64(kind):
    from ragmeup_b200.encoder import BertEncoder
    cfg, w, lm = mg.model(kind)
    enc = BertEncoder(cfg, w, with_head=False)
    L = _lib()
    _rc(L.lib().rmu_decoder_set_lm_head(enc._h, lm.ctypes.data), "lm_head")
    _dequantize(*_quantize(torch.zeros(64, dtype=torch.float16, device="cuda")))   # loads the NF4 kernels' module
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    _convert(enc)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    peak, delta = C.c_int64(), C.c_int64()
    _rc(L.lib().rmu_debug_nf4_conversion(enc._h, C.byref(peak), C.byref(delta)), "conversion")
    assert peak.value <= 0 and delta.value == _handle_bytes(cfg) < 0
    assert free1 >= free0                      # the driver sees no growth (small frees stay in its 2 MB pages)
    assert L.lib().rmu_decoder_quantize_nf4(enc._h, None) == -1 and b"already" in L.lib().rmu_last_error()
    wq = _nf4_weights(w)
    qk = kind == "qwen3"
    rng = np.random.default_rng(11)
    for T in (1, 40, 300):
        ids = rng.integers(0, cfg.vocab_size, T).tolist()
        N = 8
        logits = np.zeros((N, cfg.vocab_size), np.float32)
        rc, got = _generate(enc, ids, _sampling(), 0, N, logits)
        assert rc == 0 and len(got) == N
        ref0 = gref.logits(wq, lm, cfg, ids, qk)
        assert np.abs(logits[0] - ref0).max() <= 2e-5 * np.abs(ref0).max()
        for t in range(N):
            ref = gref.logits(wq, lm, cfg, ids + got[:t], qk)
            top2 = np.sort(ref)[-2:]
            assert np.abs(logits[t] - ref).max() <= 1e-4 * np.abs(ref).max(), t
            if top2[1] - top2[0] > 1e-4 * np.abs(ref).max():
                assert got[t] == int(np.argmax(ref)), (T, t)
            else:
                break
    # a sampled run repeats bit for bit
    s = _sampling(True, 0.8, 40, 0.9, 1.1)
    ids = rng.integers(0, cfg.vocab_size, 50).tolist()
    a = np.zeros((12, cfg.vocab_size), np.float32)
    b = np.zeros_like(a)
    ra, ta = _generate(enc, ids, s, 1234, 12, a)
    rb, tb = _generate(enc, ids, s, 1234, 12, b)
    assert ra == rb == 0 and ta == tb and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_conversion_refuses_an_encoder():
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import PRESETS, synthetic_qwen3_weights
    cfg = PRESETS["tiny-qwen3"][0]
    enc = BertEncoder(cfg, synthetic_qwen3_weights(cfg, seed=1, with_head=True), with_head=True)   # a reranker
    assert _lib().lib().rmu_decoder_quantize_nf4(enc._h, None) == -1
    assert b"rmu_encoder_create_qwen3 without a head" in _lib().lib().rmu_last_error()


def _oracle_mass(w, cfg, ids, spans, qk):
    W = {k: torch.as_tensor(v, dtype=torch.float64, device="cuda") for k, v in w.items()}
    A = da.last_attention(W, cfg, ids, qk_norm=qk)
    return torch.stack([torch.stack([A[:, a0:a1, b0:b1].sum() for b0, b1 in spans]) for a0, a1 in spans]).cpu().numpy()


@pytest.mark.parametrize("name", ["synthetic:tiny-llama", "synthetic:tiny-qwen3"])
def test_span_mass_and_sharing(name, monkeypatch):
    from ragmeup_b200 import provenance
    from ragmeup_b200.weights import resolve_decoder
    monkeypatch.setattr(provenance, "_DECODERS", {})
    monkeypatch.setenv("RMU_DECODER_WEIGHTS", "nf4")
    dec = provenance._decoder(name)
    assert dec.weights == "nf4" and provenance._decoder(name) is dec
    monkeypatch.delenv("RMU_DECODER_WEIGHTS")
    split = provenance._decoder(name)
    assert split is not dec and split.weights == "split"
    cfg, w = resolve_decoder(name)
    qk = "qwen3" in name
    ids = np.random.default_rng(4).integers(0, cfg.vocab_size, 400).tolist()
    spans = [(0, 400), (10, 120), (120, 300), (300, 399)]
    size = np.array([e - s for s, e in spans], np.float64)
    got_q, got_s = dec.span_mass(ids, spans), split.span_mass(ids, spans)
    want_q, want_s = _oracle_mass(_nf4_weights(w), cfg, ids, spans, qk), _oracle_mass(w, cfg, ids, spans, qk)
    tol = 1e-4 * cfg.heads * size[:, None]
    assert (np.abs(got_q - want_q) <= tol).all() and (np.abs(got_s - want_s) <= tol).all()
    assert np.abs(want_q - want_s).max() > np.abs(got_q - want_q).max()   # the two handles give their own results
