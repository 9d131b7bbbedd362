"""GPU: the encoder kernels one at a time (E1 split GEMM, E2 attention, E3 LayerNorm) through the rmu_debug_* entry
points, against the float64 references of oracle/encoder_kernels_ref.py, at the grids and shapes where the kernels
go wrong: several tiles per CTA on both consumer warpgroups, K-block counts that are not multiples of the 3-stage
ring, ragged last row blocks, key super-blocks, sequence boundaries.

Error unit u = 2^-24 (fp32 round-to-nearest).  Every bound is c * u * (the magnitude the rounding scales with), with
c stated once per kernel and derived next to it; the measured worst ratio |err| / (u * magnitude) is printed (-s).
"""
import math

import numpy as np
import pytest
import torch

from oracle import encoder_kernels_ref as ref

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
SENT16 = 0x7E5A                  # fp16 NaN payload in the rows past M / T: any write to them shows
SENT32 = -1234.5678


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _dev(planes):
    return tuple(torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in planes)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _sentinel16(rows, cols):
    return torch.full((rows, cols), SENT16, dtype=torch.int16, device="cuda").view(torch.float16)


def _split_ok(hi, lo):
    """the planes are a round-to-nearest split: hi finite, |lo| <= half an fp16 ulp of hi"""
    hi64 = hi.to(torch.float64)
    assert torch.isfinite(hi64).all()
    _, e = torch.frexp(hi64)                                   # |hi| in [2^(e-1), 2^e)
    ulp = torch.exp2(torch.clamp(e - 11, min=-24).to(torch.float64))
    bad = lo.to(torch.float64).abs() > 0.5 * ulp
    if bad.any():
        ij = bad.nonzero()[:8].tolist()
        pytest.fail("lo exceeds half an ulp of hi at (row, col, hi bits, lo bits) " + str(
            [(r, c, hex(int(hi[r, c].view(torch.int16)) & 0xFFFF), hex(int(lo[r, c].view(torch.int16)) & 0xFFFF))
             for r, c in ij]))


def _split_err(v):
    """|hi + lo - v| of an ideal split of v: lo carries v - hi to 11 bits (2^-22 |v|) or to the subnormal step"""
    return 2.0 ** -22 * v.abs() + 2.0 ** -25


# ----------------------------------------------------------------------------------------------------- E1
# c_gemm: the products are exact (fp16 x fp16 fits fp32), but the tensor core adds each k16 step's products to the
# fp32 accumulator with its own alignment and rounding toward zero (as measured for earlier tensor cores by Fasi et
# al., "Numerical behavior of NVIDIA tensor cores", PeerJ CS 2021), so the errors of the 3K/16 steps of one element
# do not cancel: each loses up to an ulp of a partial sum that grows as sqrt(k) for random-signed terms, which sums to
# ~0.4 u sqrt(K) S.  The epilogue adds a few roundings relative to S + |bias| + |res|.  So
# |err| <= c * u * sqrt(K) * (S + |bias| + |res|) with c = 2; the H100 measures at most 0.6 (DESIGN.md section 2).  A
# kernel that drops the lo*hi or hi*lo products is off by ~2^-12 |a||w| sqrt(K), ~5000 / sqrt(K) u S.
C_GEMM = 2.0
GELU_SLOPE = 1.13                 # max |gelu'(x)|: the accumulation error passes GELU scaled by at most this
ERF_ABS = 1.5e-7                  # Abramowitz & Stegun 7.1.26 (erf_as): |gelu error| <= 0.5 |x| * 1.5e-7 * 2 margin


def _gemm(mode, a, w, bias, res, M, qcols, qscale, max_ctas, a_rows):
    """run E1; returns float64 [M, N] (joined planes for split modes) and checks the rows past M are untouched"""
    lib = _lib()
    N = w[0].shape[0]
    pad = 8
    f32 = mode in (ref.GEMM_BIAS_F32, ref.GEMM_BIAS_RESID_F32)
    out = torch.full((M + pad, N), SENT32, dtype=torch.float32, device="cuda") if f32 else None
    oh, ol = (None, None) if f32 else (_sentinel16(M + pad, N), _sentinel16(M + pad, N))
    rc = lib.lib().rmu_debug_gemm(mode, _ptr(a[0]), _ptr(a[1]), a_rows, _ptr(w[0]), _ptr(w[1]), M, N, a[0].shape[1],
                                  _ptr(bias), _ptr(res[0]) if res else None, _ptr(res[1]) if res else None, qcols,
                                  qscale, max_ctas, _ptr(out), _ptr(oh), _ptr(ol), lib.stream_ptr())
    lib.check(rc, "rmu_debug_gemm")
    torch.cuda.synchronize()
    if f32:
        assert (out[M:] == SENT32).all(), "E1 wrote rows past M"
        return out[:M].clone(), None
    assert (oh[M:].view(torch.int16) == SENT16).all() and (ol[M:].view(torch.int16) == SENT16).all(), "E1 wrote rows past M"
    return oh[:M].clone(), ol[:M].clone()


# (mode, M, N, K, a_scale, w_scale, qcols, grids): K blocks 1..48 (1, 2, 4 ... are not multiples of the 3-stage ring),
# ragged and exact row blocks, 1 / 2 / 3 CTAs (all tiles alternating between the two consumer warpgroups of a CTA,
# odd and even tile counts per CTA) and the default grid, which for M = 4097, N = 2304 has 594 tiles on the SMs.
GEMM_CASES = [
    (0, 1, 384, 64, 1.0, 1.0, 0, (1, 2, 0)),             # 3 tiles, 1 K block
    (1, 127, 384, 128, 1.0, 0.02, 0, (1, 2, 3, 0)),      # 3 tiles, 2 K blocks
    (2, 128, 1152, 192, 16.0, 0.02, 0, (1, 2, 3, 0)),     # 9 tiles (5 + 4 on two CTAs), 3 K blocks
    (3, 129, 1152, 384, 1.0, 0.02, 384, (1, 2, 3, 0)),    # QKV of H = 384: 18 tiles, 6 K blocks, q-scale at N / 3
    (0, 1000, 1536, 256, 1e-3, 1e-3, 0, (1, 3, 0)),       # lo planes subnormal, 96 tiles, 4 K blocks
    (1, 1000, 1536, 384, 1.0, 1.0, 0, (3, 0)),            # FFN-in of MiniLM
    (2, 4097, 384, 1536, 1.0, 0.02, 0, (2, 0)),           # FFN-out of MiniLM, 24 K blocks
    (3, 4097, 2304, 768, 1.0, 0.02, 768, (3, 0)),         # QKV of bge-base: 594 tiles > SMs, 12 K blocks
    (2, 1000, 768, 3072, 1.0, 0.02, 0, (1, 0)),           # FFN-out of bge-base, 48 K blocks
    (0, 129, 128, 3072, 16.0, 1e-3, 0, (1, 0)),
    (1, 1, 1536, 64, 16.0, 1.0, 0, (2, 0)),               # large GELU arguments
    (3, 127, 384, 128, 1.0, 1.0, 0, (2, 0)),              # q-scale on no column
    (3, 127, 384, 128, 1.0, 1.0, 384, (2, 0)),            # q-scale on every column
    (3, 130, 384, 320, 1.0, 1.0, 128, (1, 0)),            # q-scale boundary at a tile edge, 5 K blocks
]


@pytest.mark.parametrize("mode,M,N,K,a_scale,w_scale,qcols,grids", GEMM_CASES)
def test_gemm_matches_float64(cuda, mode, M, N, K, a_scale, w_scale, qcols, grids):
    rng = np.random.default_rng(1000 * mode + M + N + K)
    a_rows = (M + 127) // 128 * 128 + 64                 # A's map covers more rows than M, as the activation buffers do
    a32 = np.full((a_rows, K), np.nan, np.float32)       # rows past M hold NaN: they must never reach the output
    a32[:M] = a_scale * rng.standard_normal((M, K))
    a = _dev(ref.split_f16(a32))
    w = _dev(ref.split_f16((w_scale * rng.standard_normal((N, K))).astype(np.float32)))
    bias = torch.from_numpy((0.5 * rng.standard_normal(N)).astype(np.float32)).cuda()
    res = _dev(ref.split_f16(rng.standard_normal((M, N)).astype(np.float32))) if mode == ref.GEMM_BIAS_RESID_F32 else None
    qscale = 1.0 / math.sqrt(64) * 1.4426950408889634
    outs = [_gemm(mode, a, w, bias, res, M, qcols, qscale, g, a_rows) for g in grids]
    outs.append(_gemm(mode, a, w, bias, res, M, qcols, qscale, grids[0], a_rows))      # a repeated launch
    # the per-element sum order does not depend on which CTA / warpgroup ran the tile: any difference is a race or
    # a stale ring stage; name the tiles that differ
    first = outs[0]
    for g, o in zip(list(grids) + [grids[0]], outs):
        for p0, p1 in zip(first, o):
            if p0 is None:
                continue
            same = p0.view(torch.int16 if p0.dtype == torch.float16 else torch.int32) == \
                p1.view(torch.int16 if p1.dtype == torch.float16 else torch.int32)
            if not same.all():
                bad = (~same).nonzero()
                tiles = sorted({(int(r) // 128, int(c) // 128) for r, c in bad[:4096].tolist()})
                pytest.fail(f"max_ctas={g} differs from max_ctas={grids[0]} in (row block, col block) tiles {tiles[:16]}")
    want, x, S = ref.gemm_ref(mode, a[0][:M], a[1][:M], w[0], w[1], bias, *(res or (None, None)), qcols=qcols,
                              qscale=qscale)
    if first[1] is None:
        got = first[0].to(torch.float64)
    else:
        _split_ok(*first)
        got = first[0].to(torch.float64) + first[1].to(torch.float64)
    assert torch.isfinite(got).all(), "rows below M must be finite"
    mag = S + bias.to(torch.float64).abs()[None, :]
    if res is not None:
        mag = mag + (res[0].to(torch.float64) + res[1].to(torch.float64)).abs()
    if mode == ref.GEMM_BIAS_GELU_SPLIT:
        mag = GELU_SLOPE * mag
    if mode == ref.GEMM_BIAS_SPLIT_QSCALE:
        sc = torch.ones(N, dtype=torch.float64, device="cuda")
        sc[:qcols] = float(np.float32(qscale))
        mag = mag * sc[None, :]
    err = (got - want).abs()
    extra = torch.zeros_like(err)
    if mode == ref.GEMM_BIAS_GELU_SPLIT:
        extra += 2 * ERF_ABS * 0.5 * x.abs()
    if first[1] is not None:
        extra += _split_err(want)
    ratio = float(((err - extra).clamp(min=0) / (U * math.sqrt(K) * mag)).max())
    print(f"\nE1 mode={mode} M={M} N={N} K={K} scales=({a_scale},{w_scale}) qcols={qcols}: "
          f"worst |err|/(u sqrt(K) S) = {ratio:.3g}")
    assert ratio <= C_GEMM, f"E1 error {ratio:.3g} u sqrt(K) S exceeds {C_GEMM}"


# ----------------------------------------------------------------------------------------------------- E2
# c_att, in units of 2^-22 max|V| (per sequence and head): the scores are fp32 sums of d_h three-term products, off
# by a few u * sum_d |q_d k_d| = A (log2 units), which moves each p = 2^s by ln2 * that; P is split to 22 bits,
# ex2.approx is good to 2 ulp, and P V accumulates in fp32 with the lo * lo term dropped (2^-22).  Each of these
# moves ctx by at most (relative error) * max|V| (ctx is a convex combination of V rows), so
# |err| <= c * 2^-22 * max|V| * (1 + A) with c = 8.  A kernel that drops ql * kh moves scores by ~2^-12 |q||k|.
C_ATT = 8.0
LENS = [1, 2, 15, 16, 17, 31, 32, 33, 159, 160, 161, 255, 256, 257, 300, 511, 512]


def _attention(qkv, cu, H, heads, max_seqlen, warps):
    lib = _lib()
    T = qkv[0].shape[0]
    pad = 8
    ch, cl = _sentinel16(T + pad, H), _sentinel16(T + pad, H)
    cu_d = torch.from_numpy(np.asarray(cu, np.int32)).cuda()
    rc = lib.lib().rmu_debug_attention(_ptr(qkv[0]), _ptr(qkv[1]), _ptr(cu_d), len(cu) - 1, H, heads, max_seqlen,
                                       warps, _ptr(ch), _ptr(cl), lib.stream_ptr())
    lib.check(rc, "rmu_debug_attention")
    torch.cuda.synchronize()
    assert (ch[T:].view(torch.int16) == SENT16).all() and (cl[T:].view(torch.int16) == SENT16).all(), "E2 wrote rows past T"
    return ch[:T].clone(), cl[:T].clone()


def _make_qkv(rng, lens, H, heads, kind):
    """float32 [T, 3H], q pre-scaled by log2(e) / sqrt(d_h) as the QKV epilogue leaves it.  Returns (qkv, cu, checked
    sequence ids)."""
    dh = H // heads
    if kind == "poison":
        # every checked sequence sits between two poison sequences whose V is 1e4 and whose keys align with the
        # queries of the checked ones: a key read across a cu boundary or past a sequence end dominates its softmax
        full = []
        for n in lens:
            full += [int(rng.integers(20, 90)), n]
        full.append(64)
        checked = list(range(1, len(full), 2))
    else:
        full, checked = list(lens), list(range(len(lens)))
    cu = np.r_[0, np.cumsum(full)].astype(np.int64)
    T = int(cu[-1])
    q = rng.standard_normal((T, H))
    k = rng.standard_normal((T, H))
    v = rng.standard_normal((T, H))
    if kind == "peaked":                       # scores spread over about +-60 in log2 units
        q *= 20.0 / math.log2(math.e)
    elif kind == "uniform":                    # all keys of a sequence equal: ctx = mean of V
        for b in range(len(full)):
            k[cu[b]:cu[b + 1]] = k[cu[b]]
    elif kind == "poison":
        q += 1.5                               # queries share the all-ones direction
        for b in range(0, len(full), 2):
            k[cu[b]:cu[b + 1]] = 6.0
            v[cu[b]:cu[b + 1]] = 1e4
    q *= math.log2(math.e) / math.sqrt(dh)
    return np.concatenate([q, k, v], 1).astype(np.float32), cu, checked


ATT_CASES = [
    # (H, heads, kind, lens, max_seqlen or None = max(lens), warps)
    (384, 12, "random", LENS, None, (10, 5)),
    (384, 6, "random", LENS, None, (10,)),
    (768, 24, "random", LENS, None, (10, 5)),
    (768, 12, "random", LENS, None, (10,)),
    (384, 12, "peaked", LENS, None, (10, 5)),
    (768, 12, "peaked", LENS, None, (10,)),
    (384, 12, "uniform", LENS, None, (10, 5)),
    (768, 12, "uniform", LENS, None, (10,)),
    (384, 12, "poison", LENS, None, (10, 5)),
    (768, 12, "poison", LENS, None, (10,)),
    (384, 12, "random", [256], 256, (10, 5)),           # the whole sequence resident, no key super-block
    (384, 12, "random", [257], 257, (10, 5)),           # one key past the first super-block
    (768, 12, "random", [256], 256, (10,)),
    (768, 12, "random", [257], 257, (10,)),
]


@pytest.mark.parametrize("H,heads,kind,lens,max_seqlen,warps", ATT_CASES)
def test_attention_matches_float64(cuda, H, heads, kind, lens, max_seqlen, warps):
    rng = np.random.default_rng(H + heads + len(lens) + sum(map(ord, kind)))
    qkv32, cu, checked = _make_qkv(rng, lens, H, heads, kind)
    qkv = _dev(ref.split_f16(qkv32))
    ms = max_seqlen or int(np.diff(cu).max())
    outs = [_attention(qkv, cu, H, heads, ms, w) for w in warps]
    for w, o in zip(warps[1:], outs[1:]):            # each warp's arithmetic is the same whatever the CTA's height
        assert torch.equal(o[0].view(torch.int16), outs[0][0].view(torch.int16)) and \
            torch.equal(o[1].view(torch.int16), outs[0][1].view(torch.int16)), f"{w} warps differ from {warps[0]}"
    ch, cl = outs[0]
    _split_ok(ch, cl)
    got = ch.to(torch.float64) + cl.to(torch.float64)
    want, A = ref.attention_ref(qkv[0], qkv[1], cu, heads)
    dh = H // heads
    v = qkv[0][:, 2 * H:].to(torch.float64) + qkv[1][:, 2 * H:].to(torch.float64)
    worst = 0.0
    for b in checked:
        t0, t1 = int(cu[b]), int(cu[b + 1])
        vmax = v[t0:t1].abs().view(t1 - t0, heads, dh).amax((0, 2))                     # per head
        bound = 2.0 ** -22 * vmax[None, :, None] * (1 + A[t0:t1, :, None])
        err = (got[t0:t1] - want[t0:t1]).abs().view(t1 - t0, heads, dh)
        worst = max(worst, float((err / bound).max()))
    print(f"\nE2 H={H} heads={heads} {kind} lens={len(lens)} warps={warps}: worst |err|/(2^-22 max|V| (1+A)) = {worst:.3g}")
    assert worst <= C_ATT, f"E2 error {worst:.3g} exceeds {C_ATT}"


# ----------------------------------------------------------------------------------------------------- E3
# c_ln: the mean is an fp32 sum of H values (per lane, then a shuffle tree), off by a few u * max|x|; it moves xhat
# by that over sigma and the variance by twice that relative, so with the roundings of d, the variance sum, rsqrt and
# the affine map, |err| <= c * u * (|gamma| (1 + |xhat|) (1 + max|x| / sigma) + |beta|) with c = 16.  The split of y
# adds its own 2^-22 |y|.  A one-pass variance E[x^2] - mean^2 loses (max|x| / sigma)^2 u relative on the offset rows.
C_LN = 16.0


def _layernorm(x, g, b, eps):
    lib = _lib()
    T, H = x.shape
    pad = 8
    oh, ol = _sentinel16(T + pad, H), _sentinel16(T + pad, H)
    rc = lib.lib().rmu_debug_layernorm(_ptr(x), T, H, _ptr(g), _ptr(b), eps, _ptr(oh), _ptr(ol), lib.stream_ptr())
    lib.check(rc, "rmu_debug_layernorm")
    torch.cuda.synchronize()
    assert (oh[T:].view(torch.int16) == SENT16).all() and (ol[T:].view(torch.int16) == SENT16).all(), "E3 wrote rows past T"
    return oh[:T].clone(), ol[:T].clone()


def _ln_rows(rng, T, H):
    """rows cycling through: random, offset 1e3 + N(0, 1), constant (exactly summable, so mean == value), variance
    ~1e-12, magnitude 1e4.  Returns (x, constant-row mask)."""
    x = np.empty((T, H), np.float32)
    const = np.zeros(T, bool)
    for t in range(T):
        kind = t % 5
        if kind == 0:
            x[t] = rng.standard_normal(H)
        elif kind == 1:
            x[t] = 1e3 + rng.standard_normal(H)
        elif kind == 2:
            x[t] = float(rng.integers(-64, 64)) / 8.0
            const[t] = True
        elif kind == 3:
            x[t] = 1e-6 * rng.standard_normal(H)
        else:
            x[t] = 1e4 * rng.standard_normal(H)
    return x, const


@pytest.mark.parametrize("H", [128, 384, 768, 1024])
@pytest.mark.parametrize("T", [1, 7, 9, 1001])
@pytest.mark.parametrize("eps", [1e-12, 1e-5])
def test_layernorm_matches_float64(cuda, H, T, eps):
    rng = np.random.default_rng(H * 7 + T)
    x32, const = _ln_rows(rng, T, H)
    g32 = (1.0 + 0.2 * rng.standard_normal(H)).astype(np.float32)
    b32 = (0.2 * rng.standard_normal(H)).astype(np.float32)
    x, g, b = (torch.from_numpy(t).cuda() for t in (x32, g32, b32))
    oh, ol = _layernorm(x, g, b, eps)
    _split_ok(oh, ol)
    got = oh.to(torch.float64) + ol.to(torch.float64)
    want, xhat, sigma = ref.layernorm_ref(x, g, b, eps)
    # a constant row is exactly beta (d = 0 exactly), planes included
    bh, bl = ref.split_f16(b32)
    cm = torch.from_numpy(const).cuda()
    if const.any():
        assert torch.equal(oh[cm].view(torch.int16), torch.from_numpy(bh.view(np.int16)).cuda().expand(int(const.sum()), H))
        assert torch.equal(ol[cm].view(torch.int16), torch.from_numpy(bl.view(np.int16)).cuda().expand(int(const.sum()), H))
    mx = x.to(torch.float64).abs().amax(1, keepdim=True)
    mag = g.to(torch.float64).abs()[None, :] * (1 + xhat.abs()) * (1 + mx / sigma) + b.to(torch.float64).abs()[None, :]
    ratio = float((((got - want).abs() - _split_err(want)).clamp(min=0) / (U * mag)).max())
    print(f"\nE3 H={H} T={T} eps={eps}: worst |err|/(u*mag) = {ratio:.3g}")
    assert ratio <= C_LN, f"E3 error {ratio:.3g} exceeds {C_LN}"
