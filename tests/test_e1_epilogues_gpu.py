"""GPU: E1's model-family epilogues one at a time against float64 (oracle/encoder_kernels_ref.py ``gemm_ref``), with the
harness of tests/test_encoder_kernels_gpu.py's GEMM_CASES: ModernBERT's rotary q / k (mode 4), GeGLU (mode 5) and fp32
residual (mode 6, in place and not), Qwen3 / Llama's SwiGLU (mode 7), and modes 0 / 6 / 7 at the shapes one decode step
runs (M = 1: the QKV projection, o_proj and down_proj, gate / up and the LM heads of Llama-3 and Qwen3).

Every case: A's rows past M hold NaN (mode 7: NaN and values whose outputs overflow fp16), the output rows past M hold
a sentinel, the grids listed and a repeated launch give the same bits, split outputs are round-to-nearest splits, and the
error against float64 stays within c * (the bound unit derived next to each constant).  The worst ratio is printed (-s).
References run in column chunks, so no float64 temporary passes about a GB.
"""
import math

import numpy as np
import pytest
import torch

from oracle import encoder_kernels_ref as ref
from ragmeup_b200.weights import rope_table
from test_encoder_kernels_gpu import C_GEMM, ERF_ABS, GELU_SLOPE, SENT16, SENT32, U, _sentinel16, _split_err, _split_ok

pytestmark = pytest.mark.gpu

# Each bound is c * u * sqrt(K) * (a magnitude per output) + terms that do not grow with K.  The accumulator of an output
# column is off by at most e = C_GEMM * u * sqrt(K) * (S + |b|) (S = sum_k |a w|; tests/test_encoder_kernels_gpu.py
# derives it; the H100 measures at most 0.6 up to K = 3072).  Per epilogue, in units of u * sqrt(K):
#
# * rotary (mode 4): out_c = (x_c cos - x_p sin) * sc, p the partner column in the head, so the accumulators contribute
#   ((S_c + |b_c|) |cos| + (S_p + |b_p|) |sin|) * |sc|.  The two products, the sum and the q-scale product round four
#   times against at most the same magnitude: 4 u, which is 4 / sqrt(K) <= 0.5 of the unit for K >= 64.
C_ROPE = C_GEMM + 0.5
# * GeGLU (mode 5): out = gelu(in) * gate.  |gelu'| <= GELU_SLOPE, so 1.13 (S_in + |b_in|) |gate| + |gelu(in)| (S_gate +
#   |b_gate|).  Independent of K: erf_as is within 1.5e-7 of erf, which moves gelu by 0.5 |in| 1.5e-7 (ERF_ABS |in| |gate|
#   keeps a factor 2); the fp32 gelu (the argument's scaling, 1 - p t exp, 1 + erf, 0.5 x (..)) rounds against at most 2
#   in absolute erf units, so 0.5 |in| * 4 u; the product with the gate adds u |out|; the split 2^-22 |out|.
C_GEGLU = C_GEMM
# * SwiGLU (mode 7): out = silu(in) * gate, max |silu'| = 1.0998: 1.1 (S_in + |b_in|) |gate| + |silu(in)| (S_gate +
#   |b_gate|).  Independent of K: expf (2 ulp), 1 + e, the division and the product are 5 u of |out|; the split
#   2^-22 |out|.
C_SWIGLU = C_GEMM
SILU_SLOPE = 1.1
# * fp32 residual (mode 6): out = (acc + b) + res: the accumulator's (S + |b|), then the add of res rounds against |out|
#   (u |out|; 2 u kept).  At |res| = 1e5 that second term is the one that matters.
C_RESF32 = C_GEMM
REF_CHUNK = 1 << 25                # float64 elements of one W chunk in the reference (256 MB)
PAD = 8                            # output rows past M that must keep the sentinel


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def _split(x32):
    hi = x32.half()
    return hi, (x32 - hi.float()).half()


def _rand_planes(rows, cols, scale, gen, chunk=1 << 26):
    """(hi, lo) planes [rows, cols] of scale * N(0, 1), generated on the device in row chunks (the LM heads' float32
    weights alone would be 2 GB)"""
    hi = torch.empty((rows, cols), dtype=torch.float16, device="cuda")
    lo = torch.empty_like(hi)
    step = max(1, chunk // cols)
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        x = torch.randn((r1 - r0, cols), device="cuda", generator=gen) * scale
        hi[r0:r1], lo[r0:r1] = _split(x)
    return hi, lo


def _run(mode, a, w, bias, M, grid, res=None, out=None, rope=None, qcols=0, qscale=1.0, flag=None):
    """one E1 launch; returns the output rows [:M] (fp32, or the (hi, lo) planes) after checking the rows past M kept
    their sentinel.  Mode 6: `out` is the fp32 buffer [M + PAD, N] (may be `res` itself)."""
    L = _lib()
    N, K = w[0].shape
    a_rows = a[0].shape[0]
    oh = ol = None
    if mode in (ref.GEMM_BIAS_F32, ref.GEMM_BIAS_RESF32_F32):
        if out is None:
            out = torch.full((M + PAD, N), SENT32, dtype=torch.float32, device="cuda")
    else:
        cols = N // 2 if mode in ref.GATED_MODES else N
        oh, ol = _sentinel16(M + PAD, cols), _sentinel16(M + PAD, cols)
    if mode in (ref.GEMM_BIAS_F32, ref.GEMM_BIAS_SPLIT_QSCALE):
        rc = L.lib().rmu_debug_gemm(mode, _ptr(a[0]), _ptr(a[1]), a_rows, _ptr(w[0]), _ptr(w[1]), M, N, K, _ptr(bias),
                                    None, None, qcols, qscale, grid, _ptr(out), _ptr(oh), _ptr(ol), L.stream_ptr())
    elif mode == ref.GEMM_BIAS_SWIGLU_SPLIT:
        rc = L.lib().rmu_debug_gemm_swiglu(_ptr(a[0]), _ptr(a[1]), a_rows, _ptr(w[0]), _ptr(w[1]), M, N, K, _ptr(bias),
                                           grid, _ptr(oh), _ptr(ol), _ptr(flag), L.stream_ptr())
    else:
        pos, cos, sin, hd = rope or (None, None, None, 64)
        rc = L.lib().rmu_debug_gemm_ex(mode, _ptr(a[0]), _ptr(a[1]), a_rows, _ptr(w[0]), _ptr(w[1]), M, N, K,
                                       _ptr(bias), _ptr(res), qcols, qscale, _ptr(pos), _ptr(cos), _ptr(sin),
                                       0 if cos is None else cos.shape[0], hd, grid, _ptr(out), _ptr(oh), _ptr(ol),
                                       L.stream_ptr())
    L.check(rc, f"E1 mode {mode}")
    torch.cuda.synchronize()
    if out is not None:
        assert (out[M:] == SENT32).all(), "E1 wrote rows past M"
        return (out[:M].clone(),)
    assert (oh[M:].view(torch.int16) == SENT16).all() and (ol[M:].view(torch.int16) == SENT16).all(), \
        "E1 wrote rows past M"
    return oh[:M].clone(), ol[:M].clone()


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _same_bits(first, other, what, col_tile):
    """fail naming the (row block, col block) tiles where `other` differs from `first`"""
    for p0, p1 in zip(first, other):
        same = _bits(p0) == _bits(p1)
        if not same.all():
            bad = (~same).nonzero()
            tiles = sorted({(int(r) // 128, int(c) // col_tile) for r, c in bad[:4096].tolist()})
            pytest.fail(f"{what}: (row block, col block) tiles {tiles[:16]} differ")


def _joined(outs):
    if len(outs) == 1:
        return outs[0].to(torch.float64)
    _split_ok(*outs)
    return outs[0].to(torch.float64) + outs[1].to(torch.float64)


def _worst_ratio(mode, got, a, w, bias, M, res=None, rope=None, qcols=0, qscale=1.0):
    """max over the outputs of (|got - want| - the K-independent terms) / (u sqrt(K) * the mode's magnitude), with the
    float64 reference in chunks of W rows (whole 128-row blocks)"""
    N, K = w[0].shape
    unit = U * math.sqrt(K)
    ah, al = a[0][:M], a[1][:M]
    gated = mode in ref.GATED_MODES
    step = N if mode == ref.GEMM_BIAS_SPLIT_ROPE else max(128, REF_CHUNK // K // 128 * 128)
    worst = 0.0
    for c0 in range(0, N, step):
        c1 = min(N, c0 + step)
        b = bias[c0:c1]
        want, x, S = ref.gemm_ref(mode, ah, al, w[0][c0:c1], w[1][c0:c1], b, qcols=qcols, qscale=qscale,
                                  res_f32=None if res is None else res[:M, c0:c1],
                                  **({} if rope is None else dict(pos=rope[0][:M], rope_cos=rope[1], rope_sin=rope[2],
                                                                  head_dim=rope[3])))
        ab = b.to(torch.float64).abs()[None, :]
        if gated:
            ab = ref.deblock(ab)
            F = (c1 - c0) // 2
            xin, xg = x[:, :F], x[:, F:]
            ein, eg = S[:, :F] + ab[:, :F], S[:, F:] + ab[:, F:]
            g = got[:, c0 // 2:c1 // 2]
            if mode == ref.GEMM_BIAS_GEGLU_SPLIT:
                act = 0.5 * xin * (1.0 + torch.special.erf(xin / math.sqrt(2.0)))
                mag = GELU_SLOPE * ein * xg.abs() + act.abs() * eg
                extra = (ERF_ABS + 4 * U) * xin.abs() * xg.abs() + 2 * U * want.abs()
            else:
                mag = SILU_SLOPE * ein * xg.abs() + (xin * torch.sigmoid(xin)).abs() * eg
                extra = 6 * U * want.abs()
            extra = extra + _split_err(want)
        elif mode == ref.GEMM_BIAS_SPLIT_ROPE:
            C, Sn = ref.rope_columns(rope[0][:M], rope[1], rope[2], N, qcols, rope[3])
            e = S + ab
            sc = torch.ones(N, dtype=torch.float64, device="cuda")
            sc[:qcols] = float(np.float32(qscale))
            mag = (e * C.abs() + ref.rope_partner(e, qcols, rope[3]) * Sn.abs()) * sc[None, :]
            g, extra = got, _split_err(want)
        else:
            mag = S + ab
            g = got[:, c0:c1]
            extra = 2 * U * want.abs() if mode == ref.GEMM_BIAS_RESF32_F32 else torch.zeros_like(want)
        assert torch.isfinite(g).all(), "rows below M must be finite"
        err = (g - want).abs()
        worst = max(worst, float(((err - extra).clamp(min=0) / (unit * mag)).max()))
    return worst


C_MODE = {ref.GEMM_BIAS_F32: C_GEMM, ref.GEMM_BIAS_SPLIT_ROPE: C_ROPE, ref.GEMM_BIAS_GEGLU_SPLIT: C_GEGLU,
          ref.GEMM_BIAS_RESF32_F32: C_RESF32, ref.GEMM_BIAS_SWIGLU_SPLIT: C_SWIGLU}

# (mode, M, N, K, grids, kind): one row at the decode shapes (Llama-3.1-8B: H = 4096, F = 14 336, 32 q / 8 kv heads;
# Qwen3-0.6B: H = 1024, F = 3072, 16 q heads of 128), ragged row blocks, 1 / 2 / 3 CTAs and the default grid (0), which
# for the LM heads puts 1002 and 1187 tiles on the SMs.
E1_CASES = [
    (4, 1, 2304, 768, (1, 2, 0), "d64"),           # one row, ModernBERT-base QKV
    (4, 127, 768, 128, (1, 2, 3, 0), "d32"),       # d_h 32: two heads per 64-column block, qcols 256
    (4, 129, 640, 192, (1, 3, 0), "q192"),         # qcols 192: the q / k boundary mid-tile, v past 3 qcols
    (4, 4097, 3072, 1024, (3, 0), "d64"),          # ModernBERT-large: 792 tiles, 16 K blocks
    (5, 1, 2304, 768, (1, 2, 0), ""),              # F = 1152
    (5, 127, 5248, 1024, (1, 2, 3, 0), ""),        # F = 2624, not a multiple of 128
    (5, 300, 5248, 128, (2, 0), "tails"),          # inputs to +-30 (erf tails), gates near 0
    (6, 1, 4096, 14336, (1, 2, 0), ""),            # Llama-8B down_proj at decode: 224 K blocks
    (6, 1, 1024, 2048, (1, 0), ""),                # Qwen3-0.6B o_proj at decode
    (6, 129, 768, 1152, (1, 2, 3, 0), "res1e5"),   # residual 1e5, past fp16's range
    (6, 4097, 1024, 3072, (3, 0), ""),             # prefill down_proj
    (7, 1, 28672, 4096, (1, 2, 0), ""),            # Llama-8B gate / up at decode: 224 tiles
    (7, 1, 6144, 1024, (1, 0), ""),                # Qwen3-0.6B gate / up at decode
    (7, 300, 768, 256, (2, 0), "gates40"),         # silu arguments to +-40 (expf tails, silu -> -0)
    (7, 4097, 6144, 1024, (3, 0), ""),             # prefill gate / up
    (0, 1, 6144, 4096, (1, 2, 0), ""),             # Llama-8B QKV at decode
    (0, 1, 128256, 4096, (1, 0), ""),              # Llama-3 LM head: 1002 tiles
    (0, 1, 151936, 1024, (3, 0), ""),              # Qwen3 LM head: 1187 tiles (odd)
]

ROPE_ROWS = 8192
HEAD_DIM = {"d64": 64, "d32": 32, "q192": 64}
QCOLS = {(768, "d32"): 256, (640, "q192"): 192}


@pytest.mark.parametrize("mode,M,N,K,grids,kind", E1_CASES)
def test_e1_epilogue_matches_float64(cuda, mode, M, N, K, grids, kind):
    gen = torch.Generator(device="cuda").manual_seed(7919 * mode + 31 * M + N + K)
    a_rows = (M + 127) // 128 * 128 + 64           # A's map covers more rows than M, as the activation buffers do
    a32 = torch.full((a_rows, K), float("nan"), device="cuda")
    a32[:M] = torch.randn((M, K), device="cuda", generator=gen)
    if mode == ref.GEMM_BIAS_SWIGLU_SPLIT:
        a32[M + 1::2] = 2e4                        # rows past M whose outputs overflow fp16 (and NaN rows between)
    a = _split(a32)
    w_scale = 1.0 / math.sqrt(K)
    w = _rand_planes(N, K, w_scale, gen)
    bias = 0.5 * torch.randn(N, device="cuda", generator=gen)
    if kind in ("tails", "gates40"):
        # tails: inputs ~ N(0, 11^2) (erf's tails) and gates ~ 1e-2; gates40: silu arguments ~ N(0, 13^2), some past -40
        s_in, s_gate = (1.0, 1e-3) if kind == "tails" else (0.83, w_scale)
        gate_rows = (torch.arange(N, device="cuda") % 128) >= 64
        w = _split(torch.randn((N, K), device="cuda", generator=gen) *
                   torch.where(gate_rows, s_gate, s_in)[:, None])
        if kind == "tails":
            bias = torch.where(gate_rows, 1e-3 * bias, bias)
    res = None
    if mode == ref.GEMM_BIAS_RESF32_F32:
        res = torch.full((M + PAD, N), SENT32, device="cuda")
        res[:M] = torch.randn((M, N), device="cuda", generator=gen) * (1e5 if kind == "res1e5" else 1.0)
    gated = mode in ref.GATED_MODES
    col_tile = 64 if gated else 128

    tables = [None]
    qcols, qscale = 0, 1.0
    if mode == ref.GEMM_BIAS_SPLIT_ROPE:
        hd = HEAD_DIM[kind]
        qcols = QCOLS.get((N, kind), N // 3)
        qscale = math.log2(math.e) / math.sqrt(hd)
        pos = torch.randint(0, ROPE_ROWS, (M,), device="cuda", generator=gen, dtype=torch.int32)
        if M >= 5:
            # rows 3 and 4 repeat rows 0 and 2 at a negative position and one past the table: they clamp to 0 and
            # ROPE_ROWS - 1, so their bits must be rows 0 and 2's
            pos[:5] = torch.tensor([0, 1, ROPE_ROWS - 1, -7, ROPE_ROWS + 13], dtype=torch.int32)
            a = tuple(p.clone() for p in a)
            for p in a:
                p[3], p[4] = p[0], p[2]
        tables = [tuple(torch.from_numpy(t).cuda() for t in rope_table(theta, hd, ROPE_ROWS))
                  for theta in (160000.0, 10000.0)]        # ModernBERT's global and local theta
    flag = torch.zeros(1, dtype=torch.int32, device="cuda") if mode == ref.GEMM_BIAS_SWIGLU_SPLIT else None

    for ti, tab in enumerate(tables):
        rope = None if tab is None else (pos, tab[0], tab[1], hd)

        def launch(g, in_place=True):
            if mode != ref.GEMM_BIAS_RESF32_F32:
                return _run(mode, a, w, bias, M, g, rope=rope, qcols=qcols, qscale=qscale, flag=flag)
            if in_place:                           # out = res: the residual is copied back before each launch
                buf = res.clone()
                return _run(mode, a, w, bias, M, g, res=buf, out=buf)
            return _run(mode, a, w, bias, M, g, res=res.clone())

        outs = [launch(g) for g in grids] + [launch(grids[0])]
        if mode == ref.GEMM_BIAS_RESF32_F32:
            outs.append(launch(grids[0], in_place=False))
        first = outs[0]
        for i, o in enumerate(outs[1:], 1):
            what = f"max_ctas={grids[i] if i < len(grids) else grids[0]}" + \
                (" (out apart from res)" if i == len(grids) + 1 else "")
            _same_bits(first, o, f"{what} differs from max_ctas={grids[0]}", col_tile)
        got = _joined(first)
        ratio = _worst_ratio(mode, got, a, w, bias, M, res=res, rope=rope, qcols=qcols, qscale=qscale)
        print(f"\nE1 mode={mode} M={M} N={N} K={K} {kind}{'' if tab is None else ' table %d' % ti}: "
              f"worst |err| / (u sqrt(K) mag) = {ratio:.3g}")
        assert ratio <= C_MODE[mode], f"E1 mode {mode} error {ratio:.3g} exceeds {C_MODE[mode]}"

        if mode == ref.GEMM_BIAS_SPLIT_ROPE:
            if M >= 5:
                for r, r0 in ((3, 0), (4, 2)):
                    assert torch.equal(_bits(first[0][r]), _bits(first[0][r0])) and \
                        torch.equal(_bits(first[1][r]), _bits(first[1][r0])), f"row {r}: position not clamped"
            # the v columns are mode 3's output bit for bit (same qscale, qcols covering q only)
            m3 = _run(ref.GEMM_BIAS_SPLIT_QSCALE, a, w, bias, M, 0, qcols=qcols, qscale=qscale)
            _same_bits(tuple(p[:, 2 * qcols:] for p in first), tuple(p[:, 2 * qcols:] for p in m3),
                       "v columns of mode 4 and mode 3", 128)
            assert float((got[:, :2 * qcols] - _joined(m3)[:, :2 * qcols]).abs().max()) > 1e-3   # q / k rotated

    if mode == ref.GEMM_BIAS_SWIGLU_SPLIT:
        # rows past M overflowed in every launch above and must not have set the flag; a row below M sets it
        assert int(flag.item()) == 0, "the range flag was set by rows past M"
        big = _split(torch.where(torch.arange(a_rows, device="cuda")[:, None] == M - 1, 300.0 * a32, a32))
        _run(mode, big, w, bias, M, grids[0], flag=flag)
        assert int(flag.item()) == 1, "an output of row M - 1 past fp16's range did not set the flag"
