"""CPU: the NF4 oracle (oracle/nf4_ref.py), the RMU_DECODER_WEIGHTS setting and the decoder handle's keying, and the
C refusals of the NF4 entry points."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

from oracle import nf4_ref as nf4

# Dettmers et al., QLoRA (2023), Appendix E
QLORA_NF4 = [-1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635,
             -0.18477343022823334, -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725,
             0.24611230194568634, 0.33791524171829224, 0.44070982933044434, 0.5626170039176941,
             0.7229568362236023, 1.0]


def test_code_table_and_thresholds():
    assert nf4.CODE.dtype == np.float32 and nf4.CODE.tolist() == np.array(QLORA_NF4, np.float32).tolist()
    t = nf4.THRESHOLDS.astype(np.float64)
    c = nf4.CODE.astype(np.float64)
    assert (c[:-1] < t).all() and (t < c[1:]).all()
    # each is the midpoint of its neighbours, to the printed digits
    assert np.abs(t - (c[:-1] + c[1:]) / 2).max() < 1e-7


def test_every_code_times_absmax_dequantises_to_itself():
    rng = np.random.default_rng(0)
    for a in np.concatenate([rng.uniform(1e-3, 60000, 50), [1.0, 65504.0, 6e-8]]).astype(np.float16):
        row = (nf4.CODE * np.float32(a)).astype(np.float16)        # every code once, four times over
        w = np.tile(row, 4)[None, :]
        codes, absmax = nf4.quantize(w)
        assert absmax[0, 0] == np.float32(a)
        if len(np.unique(row)) == 16:                                 # a subnormal absmax merges code values
            assert (nf4.unpack(codes)[0] == np.tile(np.arange(16), 4)).all(), a
        assert (nf4.dequantize(codes, absmax) == w).all()                # -0.0 may come back as 0.0


def test_absmax_element_maps_to_plus_or_minus_one():
    rng = np.random.default_rng(1)
    w = rng.standard_normal((64, 256)).astype(np.float16)
    codes, absmax = nf4.quantize(w)
    q = nf4.unpack(codes).reshape(64, 4, 64)
    blocks = w.astype(np.float32).reshape(64, 4, 64)
    at = np.abs(blocks).argmax(-1)
    top = np.take_along_axis(q, at[..., None], -1)[..., 0]
    sign = np.take_along_axis(blocks, at[..., None], -1)[..., 0] > 0
    assert (top == np.where(sign, 15, 0)).all()
    assert (absmax == np.abs(blocks).max(-1)).all()


def test_random_blocks_round_to_the_nearest_code_under_strict_greater():
    rng = np.random.default_rng(2)
    w = (rng.standard_normal((128, 512)) * rng.uniform(1e-3, 100, (128, 1))).astype(np.float16)
    codes, absmax = nf4.quantize(w)
    q = nf4.unpack(codes)
    a = np.repeat(absmax, 64, axis=1)
    x = (w.astype(np.float32) * (np.float32(1) / a)).astype(np.float32)
    # strict '>': the code is the count of thresholds below x, so x lies in (t[q - 1], t[q]]
    lo = np.concatenate([[-np.inf], nf4.THRESHOLDS])[q]
    hi = np.concatenate([nf4.THRESHOLDS, [np.inf]])[q]
    assert ((x > lo) & (x <= hi)).all()
    # away from a threshold that is the nearest code value
    d = np.abs(x[..., None].astype(np.float64) - nf4.CODE.astype(np.float64))
    clear = np.sort(d, -1)[..., 1] - np.sort(d, -1)[..., 0] > 1e-6
    assert (q[clear] == d.argmin(-1)[clear]).all() and clear.mean() > 0.99
    # a value exactly on a threshold takes the lower code
    t = nf4.THRESHOLDS[9]
    w1 = np.zeros((1, 64), np.float32)
    w1[0, 0], w1[0, 1] = 1.0, t
    c1, _ = nf4.quantize(w1.astype(np.float16))
    assert nf4.unpack(c1)[0, 1] == (10 if np.float32(np.float16(t)) > t else 9)


def test_all_zero_and_single_spike_blocks():
    w = np.zeros((2, 128), np.float16)
    w[1, 64 + 17] = np.float16(-3.5)
    codes, absmax = nf4.quantize(w)
    q = nf4.unpack(codes)
    d = nf4.dequantize(codes, absmax)
    # an all-zero block: absmax 0, every scaled value NaN, which passes no threshold: code 0, dequantised -0.0
    assert absmax[0, 0] == 0 and absmax[0, 1] == 0 and absmax[1, 0] == 0 and (q[0] == 0).all() and (q[1, :64] == 0).all()
    assert (d[0] == 0).all() and (d[1, :64] == 0).all()
    # one non-zero element: it maps to -1.0 (code 0), every zero to code 7 (0.0)
    assert absmax[1, 1] == 3.5 and q[1, 64 + 17] == 0 and (np.delete(q[1, 64:], 17) == 7).all()
    assert d[1, 64 + 17] == np.float16(-3.5) and (np.delete(d[1, 64:], 17) == 0).all()


def test_packing_is_high_nibble_first():
    a = np.float32(2.0)
    w = np.zeros((1, 64), np.float32)
    w[0, 0], w[0, 1], w[0, 63] = nf4.CODE[15] * a, nf4.CODE[3] * a, nf4.CODE[12] * a
    codes, _ = nf4.quantize(w.astype(np.float16))
    assert codes.shape == (1, 32) and codes[0, 0] == (15 << 4 | 3) and codes[0, 31] == (7 << 4 | 12)


def test_k_not_a_multiple_of_64_is_refused():
    for K in (32, 96, 100):
        with pytest.raises(ValueError, match="multiple of 64"):
            nf4.quantize(np.zeros((2, K), np.float16))
    with pytest.raises(ValueError):
        nf4.nf4_weight(np.zeros((4, 48), np.float32))


def test_fp16_cast_equals_torch_on_bf16_values():
    bits = np.arange(0, 1 << 16, dtype=np.uint32).astype(np.uint16)
    b = torch.from_numpy(bits.view(np.int16)).view(torch.bfloat16)
    f32 = b.float()
    ok = torch.isfinite(f32) & (f32.abs() < 65520)
    f32 = f32[ok]
    want = f32.to(torch.bfloat16).to(torch.float16).numpy()
    got = nf4.to_fp16(f32.numpy())
    assert (got.view(np.uint16) == want.view(np.uint16)).all()
    # the ranges that matter: fp16 subnormals and the top of the range
    sub = np.abs(f32.numpy()) < 6.1e-5
    assert sub.sum() > 1000 and (np.abs(f32.numpy()) > 65000).sum() > 0


# ------------------------------------------------------------------------------------------------------- settings
def test_decoder_weights_setting(monkeypatch):
    from ragmeup_b200 import provenance
    monkeypatch.delenv("RMU_DECODER_WEIGHTS", raising=False)
    assert provenance.decoder_weights() == "split"
    for v, want in (("nf4", "nf4"), ("NF4", "nf4"), ("split", "split"), ("", "split")):
        monkeypatch.setenv("RMU_DECODER_WEIGHTS", v)
        assert provenance.decoder_weights() == want
    for bad in ("int8", "fp4", "nf4,split"):
        monkeypatch.setenv("RMU_DECODER_WEIGHTS", bad)
        with pytest.raises(ValueError, match="RMU_DECODER_WEIGHTS"):
            provenance.decoder_weights()
    with pytest.raises(ValueError, match="weights"):
        provenance.DecoderAttention("synthetic:tiny-llama", weights="int8")


def test_decoders_keyed_by_snapshot_device_and_weights(monkeypatch):
    from ragmeup_b200 import _lib, provenance
    made = []

    class Fake:
        def __init__(self, name, device=None, weights="split"):
            made.append((name, device, weights))

    class FakeTorch:
        class cuda:
            @staticmethod
            def current_device():
                return 0

    monkeypatch.setattr(provenance, "DecoderAttention", Fake)
    monkeypatch.setattr(_lib, "require_cuda", lambda: FakeTorch)
    monkeypatch.setattr(provenance, "_DECODERS", {})
    monkeypatch.delenv("RMU_DECODER_WEIGHTS", raising=False)
    a = provenance._decoder("synthetic:tiny-llama")
    assert provenance._decoder("synthetic:tiny-llama") is a
    assert made == [("synthetic:tiny-llama", 0, "split")]              # the default builds the handle it always did
    monkeypatch.setenv("RMU_DECODER_WEIGHTS", "nf4")
    b = provenance._decoder("synthetic:tiny-llama")
    assert b is not a and provenance._decoder("synthetic:tiny-llama") is b
    assert made[-1] == ("synthetic:tiny-llama", 0, "nf4")
    assert set(provenance._DECODERS) == {("synthetic:tiny-llama", 0, "split"), ("synthetic:tiny-llama", 0, "nf4")}


# ------------------------------------------------------------------------------------------------------ C refusals
def test_nf4_entry_points_refuse_before_any_cuda_call():
    from ragmeup_b200 import _lib
    l = _lib.lib()
    p = 1 << 20                                    # stand-in device address, never touched
    assert l.rmu_decoder_quantize_nf4(None, None) == -1
    pk, dl = ctypes.c_int64(), ctypes.c_int64()
    assert l.rmu_debug_nf4_conversion(None, ctypes.byref(pk), ctypes.byref(dl)) == -1
    for q in (l.rmu_debug_nf4_quantize,):
        assert q(None, 64, p, p, None) == -1 and q(p, 64, None, p, None) == -1 and q(p, 64, p, None, None) == -1
        assert q(p, 0, p, p, None) == -1 and q(p, -64, p, p, None) == -1
        assert q(p, 96, p, p, None) == -3 and q(p, 32, p, p, None) == -3
    d = l.rmu_debug_nf4_dequantize
    assert d(None, p, 64, p, None) == -1 and d(p, None, 64, p, None) == -1 and d(p, p, 64, None, None) == -1
    assert d(p, p, 0, p, None) == -1 and d(p, p, 100, p, None) == -3

    def gemv(mode=0, N=256, K=128, x=p, res=p, out_f32=p, out_hi=p, out_lo=p, codes=p, bias=p):
        return l.rmu_debug_nf4_gemv(mode, x, x, codes, p, N, K, bias, res, out_f32, out_hi, out_lo, None, None)

    for mode in (1, 2, 3, 4, 5, -1, 8):
        assert gemv(mode) == -1, mode
    for mode in (0, 6, 7):
        assert gemv(mode, N=192) == -3 and gemv(mode, N=64) == -3          # N % 128
        assert gemv(mode, K=96) == -3 and gemv(mode, K=32) == -3           # K % 64
        assert gemv(mode, K=49152 + 64) == -3
        assert gemv(mode, x=None) == -1 and gemv(mode, codes=None) == -1 and gemv(mode, bias=None) == -1
        assert gemv(mode, N=0) == -1 and gemv(mode, K=0) == -1
    assert gemv(0, out_f32=None) == -1 and gemv(6, out_f32=None) == -1 and gemv(6, res=None) == -1
    assert gemv(7, out_hi=None) == -1 and gemv(7, out_lo=None) == -1
    assert b"nf4" in l.rmu_last_error()
