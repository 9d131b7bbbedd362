"""GPU: the encoder kernels one at a time (E1 split GEMM, E2 attention, E3 LayerNorm and embedding LayerNorm, E4
pooling and classifier head, the plane split / join) through the rmu_debug_* entry points, against the float64
references of oracle/encoder_kernels_ref.py, at the grids and shapes where the kernels go wrong: several tiles per CTA
on both consumer warpgroups, K-block counts that are not multiples of the 3-stage ring, ragged last row blocks, key
super-blocks, sequence boundaries, empty sequences, threads with no column, fp16 overflow and subnormals.

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
    (3, 1000, 3072, 1024, 1.0, 0.02, 1024, (3, 0)),       # QKV of H = 1024 (bge-large): N = 3072, 16 K blocks
    (1, 1000, 4096, 1024, 1.0, 0.02, 0, (3, 0)),          # FFN-in of H = 1024: N = 4096
    (2, 1000, 1024, 4096, 1.0, 0.02, 0, (1, 0)),          # FFN-out of H = 1024: K = 4096, 64 K blocks
    (3, 300, 2688, 896, 1.0, 0.02, 896, (2, 0)),          # QKV of H = 896: 21 tiles wide, 14 K blocks
    (1, 300, 2688, 896, 1.0, 0.02, 0, (2, 0)),            # FFN-in of H = 896, F = 2688
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


def _attention(qkv, cu, H, heads, max_seqlen):
    lib = _lib()
    T = qkv[0].shape[0]
    pad = 8
    ch, cl = _sentinel16(T + pad, H), _sentinel16(T + pad, H)
    cu_d = torch.from_numpy(np.asarray(cu, np.int32)).cuda()
    rc = lib.lib().rmu_debug_attention(_ptr(qkv[0]), _ptr(qkv[1]), _ptr(cu_d), len(cu) - 1, H, heads, max_seqlen,
                                       10, _ptr(ch), _ptr(cl), lib.stream_ptr())
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
    # (H, heads, kind, lens, max_seqlen or None = max(lens))
    (384, 12, "random", LENS, None),
    (384, 6, "random", LENS, None),
    (768, 24, "random", LENS, None),
    (768, 12, "random", LENS, None),
    (384, 12, "peaked", LENS, None),
    (768, 12, "peaked", LENS, None),
    (384, 12, "uniform", LENS, None),
    (768, 12, "uniform", LENS, None),
    (384, 12, "poison", LENS, None),
    (768, 12, "poison", LENS, None),
    (384, 12, "random", [256], 256),                    # the whole sequence resident, no key super-block
    (384, 12, "random", [257], 257),                    # one key past the first super-block
    (768, 12, "random", [256], 256),
    (768, 12, "random", [257], 257),
    (1024, 16, "random", LENS, None),                   # bge-large: d_h = 64 at the largest H
    (1024, 32, "random", LENS, None),                   # d_h = 32 at the largest H
    (128, 2, "random", LENS, None),                     # d_h = 64 at the smallest H
]


@pytest.mark.parametrize("H,heads,kind,lens,max_seqlen", ATT_CASES)
def test_attention_matches_float64(cuda, H, heads, kind, lens, max_seqlen):
    rng = np.random.default_rng(H + heads + len(lens) + sum(map(ord, kind)))
    qkv32, cu, checked = _make_qkv(rng, lens, H, heads, kind)
    qkv = _dev(ref.split_f16(qkv32))
    ms = max_seqlen or int(np.diff(cu).max())
    ch, cl = _attention(qkv, cu, H, heads, ms)
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
    print(f"\nE2 H={H} heads={heads} {kind} lens={len(lens)}: worst |err|/(2^-22 max|V| (1+A)) = {worst:.3g}")
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


@pytest.mark.parametrize("H", [128, 384, 768, 896, 1024])
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


# ----------------------------------------------------------------------------------------------- E3 embed_ln
# c_emb: the kernel sums (w + t) + p in fp32, two roundings, so its x is off by at most 2u * M with
# M = max_d (|w_d| + |t_d| + |p_d|).  To first order LayerNorm moves y_j by gamma_j / sigma * (dx_j - mean(dx) -
# xhat_j * mean(xhat dx)); with |dx| <= 2u M and mean|xhat| <= 1 that is at most 2u M |gamma_j| (2 + |xhat_j|) / sigma
# <= 4u |gamma_j| (1 + |xhat_j|) M / sigma.  The LayerNorm itself is E3's c_ln = 16 with max|x| <= M, so
# |err| <= c * u * (|gamma| (1 + |xhat|) (1 + M / sigma) + |beta|) with c = 16 + 4 = 20.  A binary search that puts the
# first token of a sequence in the previous one, or a kernel that ignores type ids, moves whole rows (~0.1 sigma).
C_EMB = 20.0
VOCAB, MAX_POS, TYPE_VOCAB = 30522, 512, 2


def _emb_tables(H, seed):
    """word rows cycle through the kinds of _ln_rows (N(0, 1), offset 1e3, constant, spread 1e-6, magnitude 1e4);
    position and type rows all differ, so a wrong row shows.  fp32 on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    kind = torch.arange(VOCAB, device="cuda") % 5
    scale = torch.tensor([1.0, 1.0, 0.0, 1e-6, 1e4], device="cuda")[kind]
    offset = torch.tensor([0.0, 1e3, 0.0, 0.0, 0.0], device="cuda")[kind] + (kind == 2) * ((torch.arange(VOCAB, device="cuda") % 128) - 64) / 8.0
    word = (torch.randn(VOCAB, H, device="cuda", generator=g) * scale[:, None] + offset[:, None]).float().contiguous()
    pos = (0.1 * torch.randn(MAX_POS, H, device="cuda", generator=g)).float().contiguous()
    typ = (0.5 * torch.randn(TYPE_VOCAB, H, device="cuda", generator=g)).float().contiguous()
    gamma = (1.0 + 0.2 * torch.randn(H, device="cuda", generator=g)).float().contiguous()
    beta = (0.2 * torch.randn(H, device="cuda", generator=g)).float().contiguous()
    return word, pos, typ, gamma, beta


def _i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()


def _embed_ln(ids, tt, cu, tabs, eps=1e-12):
    """run E3 embed_ln on int32 device ids / type ids (or None) / cu; checks the rows past T are untouched"""
    lib = _lib()
    word, pos, typ, g, b = tabs
    T, H = ids.numel(), word.shape[1]
    pad = 8
    oh, ol = _sentinel16(T + pad, H), _sentinel16(T + pad, H)
    rc = lib.lib().rmu_debug_embed_ln(_ptr(ids), _ptr(tt), _ptr(cu), cu.numel() - 1, T, H, word.shape[0], pos.shape[0],
                                      typ.shape[0], _ptr(word), _ptr(pos), _ptr(typ), _ptr(g), _ptr(b), eps, _ptr(oh),
                                      _ptr(ol), lib.stream_ptr())
    lib.check(rc, "rmu_debug_embed_ln")
    torch.cuda.synchronize()
    assert (oh[T:].view(torch.int16) == SENT16).all() and (ol[T:].view(torch.int16) == SENT16).all(), "embed_ln wrote rows past T"
    return oh[:T].clone(), ol[:T].clone()


def _emb_lens(batch, rng):
    """ragged batches: length-1 sequences, empty ones in the middle and at the end, one sequence of exactly MAX_POS
    (T = 4097), and 70 000 sequences of 0 to 3 tokens"""
    if batch == "T=1":
        return [1]
    if batch == "T=7":
        return [1, 0, 3, 0, 2, 1, 0]
    if batch == "T=9":
        return [0, 4, 0, 0, 5, 0]
    if batch == "T=4097":
        lens = [MAX_POS, 1, 0, 300, 147]
        while sum(lens) < 4097 - 200:
            lens.append(int(rng.integers(1, 200)))
        lens += [4097 - sum(lens), 0, 0]
        return lens
    assert batch == "B=70000"
    return rng.integers(0, 4, 70000).tolist()


def _same(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# H = 128 ... 1024: per_lane 4 to 32, every branch of the kernel's unrolled loops; T not a multiple of 8 tokens per block
EMB_CASES = [(H, batch) for H in (128, 256, 384, 640, 768, 896, 1024) for batch in ("T=1", "T=7", "T=9", "T=4097")] + \
    [(128, "B=70000"), (768, "B=70000")]


@pytest.mark.parametrize("H,batch", EMB_CASES)
def test_embed_ln_matches_float64(cuda, H, batch):
    rng = np.random.default_rng(H * 11 + len(batch) + ord(batch[-1]))
    lens = _emb_lens(batch, rng)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    T = int(cu[-1])
    ids = rng.integers(0, VOCAB, T)
    ids[::11] = 0
    ids[5::13] = VOCAB - 1
    tt = rng.integers(0, TYPE_VOCAB, T)
    tabs = _emb_tables(H, H + T)
    ids_d, tt_d, cu_d = _i32(ids), _i32(tt), _i32(cu)
    oh, ol = _embed_ln(ids_d, tt_d, cu_d, tabs)
    _split_ok(oh, ol)
    got = oh.to(torch.float64) + ol.to(torch.float64)
    want, xhat, sigma, M = ref.embed_ln_ref(ids_d, tt_d, cu_d, *tabs, 1e-12)
    g, b = tabs[3].to(torch.float64), tabs[4].to(torch.float64)
    mag = g.abs()[None, :] * (1 + xhat.abs()) * (1 + M / sigma) + b.abs()[None, :]
    ratio = float((((got - want).abs() - _split_err(want)).clamp(min=0) / (U * mag)).max())
    print(f"\nE3 embed_ln H={H} T={T} B={len(lens)}: worst |err|/(u*mag) = {ratio:.3g}")
    assert ratio <= C_EMB, f"embed_ln error {ratio:.3g} exceeds {C_EMB}"
    # no type ids = explicit zeros, bit for bit
    z = _embed_ln(ids_d, None, cu_d, tabs)
    assert all(_same(p, q) for p, q in zip(z, _embed_ln(ids_d, torch.zeros_like(ids_d), cu_d, tabs)))
    # a token's planes do not depend on the batch it sits in: each of a few sequences alone
    for s in sorted({0, len(lens) // 2, len(lens) - 1, int(np.argmax(lens))}):
        t0, t1 = int(cu[s]), int(cu[s + 1])
        if t1 == t0:
            continue
        ah, al = _embed_ln(ids_d[t0:t1].clone(), tt_d[t0:t1].clone(), _i32([0, t1 - t0]), tabs)
        assert _same(ah, oh[t0:t1]) and _same(al, ol[t0:t1]), f"sequence {s} alone differs from its batch"


def test_embed_ln_clamps_out_of_range_inputs(cuda):
    """ids clamp into [0, vocab), type ids into [0, type_vocab), positions to max_pos - 1 (HuggingFace raises instead):
    the clamped row, bit for bit"""
    H = 384
    tabs = _emb_tables(H, 7)
    lens = [MAX_POS + 5, 6]
    cu = _i32(np.r_[0, np.cumsum(lens)])
    T = sum(lens)
    ids = np.full(T, 1234)
    tt = np.ones(T, np.int64)
    bad_ids = [-5, VOCAB, VOCAB + 7, -(2 ** 31), 2 ** 31 - 1, 3]
    bad_tt = [-1, 2, 7, -(2 ** 31), 2 ** 31 - 1, 0]
    ids[MAX_POS + 5:] = bad_ids
    tt[MAX_POS + 5:] = bad_tt
    oh, ol = _embed_ln(_i32(ids), _i32(tt), cu, tabs)
    ch, cl = _embed_ln(_i32(np.clip(ids, 0, VOCAB - 1)), _i32(np.clip(tt, 0, TYPE_VOCAB - 1)), cu, tabs)
    assert _same(oh, ch) and _same(ol, cl)
    # the first sequence runs past max_pos with one id and type: positions max_pos - 1 .. max_pos + 4 share a row
    for t in range(MAX_POS, MAX_POS + 5):
        assert _same(oh[t], oh[MAX_POS - 1]) and _same(ol[t], ol[MAX_POS - 1])
    assert not _same(oh[MAX_POS - 2], oh[MAX_POS - 1])
    want = ref.embed_ln_ref(_i32(ids), _i32(tt), cu, *tabs, 1e-12)[0]          # the reference clamps the same way
    assert float((oh.to(torch.float64) + ol.to(torch.float64) - want).abs().max()) < 1e-3


# ---------------------------------------------------------------------------------------------------- E4 pool
# c_pool, unnormalised: hi + lo is exact in fp32 (22 significant bits), so the only roundings are the serial fp32 sum
# over S tokens, at most (S - 1) u sum_t |x_td|, and the division by S, u |m_d| <= u mean_t |x_td|: |err| <= c u P_d with
# P_d = sum_t |x_td| = S mean_t |x_td| and c = 1 (2 with second-order terms).  CLS copies a row: exact.
# c_norm: ||m||^2 is an fmaf chain over <= 4 values per thread, a 5-level shuffle tree and a serial sum of 8 warp
# partials, all of non-negative terms: at most 4 + 5 + 7 = 16 roundings, 16u relative, 8u after the square root; sqrtf,
# the reciprocal and the multiply add u each, so 11u |n_d| with n = m / ||m||.  An error dm moves n_d by at most
# (|dm_d| + |n_d| ||dm||) / ||m||.  So |err| <= c u ((P_d + |n_d| ||P||) / max(||m||, 1e-12) + |n_d|) with c = 16.
# Summing only the hi plane is off by ~2^-12 |x| per token; normalising by warp 0's partial alone, by a factor.
C_POOL = 2.0
C_NORM = 16.0
POOL_LENS = [1, 0, 2, 147, 512, 3, 4, 0]   # S = 0, 1, 2, 147, 512; [0, x, -x] sums to exactly 0; 1e-3 rows (lo subnormal)


def _pool(hi, lo, cu, mode, normalize):
    lib = _lib()
    B, H = len(cu) - 1, hi.shape[1]
    pad = 8
    out = torch.full((B + pad, H), SENT32, dtype=torch.float32, device="cuda")
    rc = lib.lib().rmu_debug_pool(_ptr(hi), _ptr(lo), _ptr(_i32(cu)), B, H, mode, int(normalize), _ptr(out), lib.stream_ptr())
    lib.check(rc, "rmu_debug_pool")
    torch.cuda.synchronize()
    assert (out[B:] == SENT32).all(), "pool wrote rows past B"
    return out[:B].clone()


def _join_dev(hi, lo):
    """rmu_debug_join_planes over whole plane tensors -> fp32, same shape"""
    lib = _lib()
    out = torch.empty(hi.shape, dtype=torch.float32, device="cuda")
    lib.check(lib.lib().rmu_debug_join_planes(_ptr(hi), _ptr(lo), hi.numel(), _ptr(out), lib.stream_ptr()),
              "rmu_debug_join_planes")
    torch.cuda.synchronize()
    return out


def _pool_planes(rng, H, mode):
    cu = np.r_[0, np.cumsum(POOL_LENS)]
    T = int(cu[-1])
    x = rng.standard_normal((T, H)).astype(np.float32)
    x[cu[6]:cu[7]] *= 1e-3
    hi, lo = ref.split_f16(x)
    c0 = cu[5]
    hi[c0], lo[c0] = 0, 0
    hi[c0 + 2], lo[c0 + 2] = -hi[c0 + 1], -lo[c0 + 1]
    if mode == 1:                                    # CLS reads the first token only: NaN everywhere else
        for b in range(len(POOL_LENS)):
            hi[cu[b] + 1:cu[b + 1]] = np.nan
            lo[cu[b] + 1:cu[b + 1]] = np.nan
    return _dev((hi, lo)), cu


@pytest.mark.parametrize("H", [128, 200, 384, 768, 1024])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("normalize", [False, True])
def test_pool_matches_float64(cuda, H, mode, normalize):
    rng = np.random.default_rng(H + 3 * mode)
    (hi, lo), cu = _pool_planes(rng, H, mode)
    got = _pool(hi, lo, cu, mode, normalize)
    assert torch.isfinite(got).all(), "NaN or inf reached the output"
    want, m, P = ref.pool_ref(hi, lo, cu, mode, normalize)
    lens = np.diff(cu)
    zero = torch.from_numpy((lens == 0) | (np.arange(len(lens)) == 5)).cuda()   # empty, and sums / CLS row exactly 0
    assert (got[zero] == 0).all(), "an empty or all-zero sequence must pool to exactly 0"
    rows = _join_dev(hi, lo)
    if not normalize:
        if mode == 1:                                # CLS copies row cu[b]
            first = torch.from_numpy(np.minimum(cu[:-1], cu[-1] - 1)).cuda()
            assert _same32(got[~zero], rows[first][~zero])
        one = torch.from_numpy(cu[:-1][lens == 1]).cuda()
        assert _same32(got[torch.from_numpy(lens == 1).cuda()], rows[one]), "S = 1 must return the row itself"
    err = (got.to(torch.float64) - want).abs()
    if normalize:
        nrm = m.norm(dim=1, keepdim=True).clamp(min=1e-12)
        n = want.abs()
        mag = (P + n * P.norm(dim=1, keepdim=True)) / nrm + n
        c = C_NORM
    else:
        mag, c = P, C_POOL
    assert (err[mag == 0] == 0).all(), "an exact copy differs"
    ratio = float((err / (U * mag)).nan_to_num(0.0, posinf=0.0).max())
    print(f"\nE4 pool H={H} mode={'cls' if mode else 'mean'} normalize={normalize}: worst |err|/(u*mag) = {ratio:.3g}")
    assert ratio <= c, f"pool error {ratio:.3g} exceeds {c}"
    # a sequence's output does not depend on its batch: each non-empty one alone, from a fresh copy of its rows
    for b in range(len(lens)):
        t0, t1 = int(cu[b]), int(cu[b + 1])
        if t1 > t0:
            alone = _pool(hi[t0:t1].clone(), lo[t0:t1].clone(), [0, t1 - t0], mode, normalize)
            assert _same32(alone[0], got[b]), f"sequence {b} alone differs from its batch"


def _same32(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ----------------------------------------------------------------------------------------------- E4 cls_head
# c_head: each pre-activation is a lane's serial fmaf chain over H/32 terms plus a 5-level shuffle tree and the bias
# add, so with k = H/32 + 6 it is off by at most dz_j = u (k A_j + |b_pj|), A_j = sum_d |W_pjd h_d|.  tanhf is good to
# 2 ulp (CUDA C Programming Guide, math functions), at most 4u |pooled_j|, and tanh' = sech^2, so to first order
# dpooled_j <= sech^2(z_j) dz_j + 4u |pooled_j| (a saturated unit passes none of dz on).  The classifier adds
# sum_j |W_cj| dpooled_j and its own u (k C_c + |b_c|), C_c = sum_j |W_cj pooled_j|.  So
# |err| <= c u (sum_j |W_cj| (sech^2(z_j) (k A_j + |b_pj|) + 4 |pooled_j|) + k C_c + |b_c|) with c = 1 to first order;
# c = 2.  The bound is a worst case over signs: the identity-pooler test below checks h_cls and tanhf to the ulp.
C_HEAD = 2.0


def _cls_head(hi, lo, cu, H, head):
    lib = _lib()
    pw, pb, cw, cb = head
    B, L = len(cu) - 1, cw.shape[0]
    pad = 8
    out = torch.full((B + pad, L), SENT32, dtype=torch.float32, device="cuda")
    rc = lib.lib().rmu_debug_cls_head(_ptr(hi), _ptr(lo), _ptr(_i32(cu)), B, H, L, _ptr(pw), _ptr(pb), _ptr(cw), _ptr(cb),
                                      _ptr(out), lib.stream_ptr())
    lib.check(rc, "rmu_debug_cls_head")
    torch.cuda.synchronize()
    assert (out[B:] == SENT32).all(), "cls_head wrote rows past B"
    return out[:B].clone()


def _nan_tail(hi, lo, rows, pad=8):
    """planes [rows + pad, H] holding (hi, lo) and NaN in the pad rows: a read past the last sequence shows as NaN"""
    H = hi.shape[1]
    h = torch.full((rows + pad, H), float("nan"), dtype=torch.float16, device="cuda")
    l = h.clone()
    h[:rows], l[:rows] = hi, lo
    return h, l


@pytest.mark.parametrize("H", [128, 384, 768, 1024])
@pytest.mark.parametrize("L", [1, 2, 9, 17])
def test_cls_head_matches_float64(cuda, H, L):
    rng = np.random.default_rng(H + L)
    B = 1000
    lens = rng.integers(1, 6, B)
    lens[B // 2] = 0                                 # an empty sequence in the middle and at the end
    lens[-1] = 0
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    T = int(cu[-1])
    # h_cls scaled 1, 0.01 and 30 in turn, and half the pooler biases +-12: pre-activations near 0, O(1) and saturated
    scale = np.array([1.0, 0.01, 30.0])[np.repeat(np.arange(B) % 3, lens)]
    x = (rng.standard_normal((T, H)) * scale[:, None]).astype(np.float32)
    hi, lo = ref.split_f16(x)
    for b in range(B):                               # the head reads the first token only: NaN everywhere else
        hi[cu[b] + 1:cu[b + 1]] = np.nan
        lo[cu[b] + 1:cu[b + 1]] = np.nan
    hi, lo = _nan_tail(*_dev((hi, lo)), T)
    pb = np.where(np.arange(H) % 2 == 0, 0.01 * rng.standard_normal(H), 12.0 * np.sign(rng.standard_normal(H)))
    head = tuple(torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in (
        rng.standard_normal((H, H)) / math.sqrt(H), pb, rng.standard_normal((L, H)) / math.sqrt(H), rng.standard_normal(L)))
    got = _cls_head(hi, lo, cu, H, head)
    assert torch.isfinite(got).all(), "NaN reached the logits (a row other than cu[b], or past T, was read)"
    want, z, pooled, A, C = ref.cls_head_ref(hi, lo, cu, *head)
    assert (z.abs() < 0.05).any() and (z.abs() > 10).any()
    k = H / 32 + 6
    pw, pb_, cw, cb = (t.to(torch.float64) for t in head)
    sech2 = 1.0 / torch.cosh(z) ** 2
    mag = (sech2 * (k * A + pb_.abs()[None, :]) + 4 * pooled.abs()) @ cw.abs().T + k * C + cb.abs()[None, :]
    ratio = float(((got.to(torch.float64) - want).abs() / (U * mag)).max())
    print(f"\nE4 cls_head H={H} labels={L}: worst |err|/(u*mag) = {ratio:.3g}")
    assert ratio <= C_HEAD, f"cls_head error {ratio:.3g} exceeds {C_HEAD}"
    # an empty sequence scores W_c tanh(b_p) + b_c, the same in the middle and at the end
    assert _same32(got[B // 2], got[-1])
    # each pair scores the same alone as in the batch of 1000 (an empty one alone reads no row at all)
    for b in (0, 1, 2, B // 2, B - 2, B - 1):
        t0, t1 = int(cu[b]), int(cu[b + 1])
        ah, al = _nan_tail(hi[t0:t1], lo[t0:t1], t1 - t0)
        assert _same32(_cls_head(ah, al, [0, t1 - t0], H, head)[0], got[b]), f"pair {b} alone differs from its batch"


@pytest.mark.parametrize("H", [128, 1024])
def test_cls_head_identity_pooler_is_tanhf_of_h(cuda, H):
    """W_p = I, b_p = 0 and classifier rows e_j: every product but one is 0 * h, so both dot products are exact and
    logit c = tanhf(h_j(c)), which the CUDA math library keeps within 2 ulp of tanh.  h = hi + lo over 0.01 .. 12,
    both signs: any loss of the lo plane (2^-12 relative) or an approximate tanh (~2^-11) is hundreds of ulp."""
    rng = np.random.default_rng(H)
    L = 17
    B = 64
    lens = rng.integers(1, 4, B)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    x = (np.sign(rng.standard_normal((cu[-1], H))) * np.exp(rng.uniform(np.log(0.01), np.log(12.0), (cu[-1], H))))
    hi, lo = _dev(ref.split_f16(x.astype(np.float32)))
    cols = rng.choice(H, L, replace=False)
    cw = np.zeros((L, H), np.float32)
    cw[np.arange(L), cols] = 1.0
    head = tuple(torch.from_numpy(a).cuda() for a in (np.eye(H, dtype=np.float32), np.zeros(H, np.float32), cw,
                                                      np.zeros(L, np.float32)))
    got = _cls_head(hi, lo, cu, H, head).cpu().numpy()
    h = (hi.to(torch.float64) + lo.to(torch.float64)).cpu().numpy()[cu[:-1]][:, cols]
    want = np.tanh(h)
    ulps = np.abs(got - want) / np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    print(f"\nE4 cls_head identity pooler H={H}: worst |tanhf(h) - tanh(h)| = {ulps.max():.3g} ulp")
    assert ulps.max() <= 2.0, f"{ulps.max():.3g} ulp from tanh(h_cls)"


# -------------------------------------------------------------------------------------------- split / join
def _split_dev(src):
    lib = _lib()
    n = src.numel()
    pad = 300
    hi, lo = _sentinel16(1, n + pad)[0], _sentinel16(1, n + pad)[0]
    lib.check(lib.lib().rmu_debug_split_planes(_ptr(src), n, _ptr(hi), _ptr(lo), lib.stream_ptr()), "rmu_debug_split_planes")
    torch.cuda.synchronize()
    assert (hi[n:].view(torch.int16) == SENT16).all() and (lo[n:].view(torch.int16) == SENT16).all(), "split wrote past n"
    return hi[:n].clone(), lo[:n].clone()


def _join_n(hi, lo):
    lib = _lib()
    n = hi.numel()
    pad = 300
    out = torch.full((n + pad,), SENT32, dtype=torch.float32, device="cuda")
    lib.check(lib.lib().rmu_debug_join_planes(_ptr(hi), _ptr(lo), n, _ptr(out), lib.stream_ptr()), "rmu_debug_join_planes")
    torch.cuda.synchronize()
    assert (out[n:] == SENT32).all(), "join wrote past n"
    return out[:n].clone()


def _bits_match(got, want, what):
    """bit-identical, except that NaN only has to be NaN (payloads differ between numpy and the device)"""
    g, w = got.cpu().numpy(), np.asarray(want)
    nan = np.isnan(w.astype(np.float64))
    assert (np.isnan(g.astype(np.float64)) == nan).all(), f"{what}: NaN placement differs"
    ui = np.uint16 if g.dtype == np.float16 else np.uint32
    bad = np.nonzero((g.view(ui) != w.view(ui)) & ~nan)[0]
    assert bad.size == 0, f"{what}: {bad.size} values differ, first at {bad[:4].tolist()}: " \
                          f"{[hex(int(v)) for v in g.view(ui)[bad[:4]]]} vs {[hex(int(v)) for v in w.view(ui)[bad[:4]]]}"


def test_split_and_join_planes_are_bit_identical_to_the_reference(cuda):
    k = np.arange(2 ** 20, dtype=np.uint64)
    sweep = (k * 4096 + k % 4096).astype(np.uint32).view(np.float32)        # one pattern in every 4096, low bits varied
    f32min = np.float32(2.0 ** -149)
    special = np.array([0.0, -0.0, f32min, -f32min, 1e-40, -3e-39, 2.0 ** -126, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26,
                        -2.0 ** -20 * 3, 2.0 ** -14, 6.1e-5, 0.1, 1.0, -2.5, 65504.0, -65504.0,
                        np.nextafter(np.float32(65520), np.float32(0)), 65520.0, -65520.0, 65536.0, 1e30, np.inf,
                        -np.inf, np.nan], np.float32)
    rng = np.random.default_rng(9)
    v = np.concatenate([sweep, special, rng.standard_normal(77).astype(np.float32)])          # n % 256 != 0
    assert v.size % 256 != 0
    hi, lo = _split_dev(torch.from_numpy(v).cuda())
    with np.errstate(over="ignore", invalid="ignore"):
        wh, wl = ref.split_f16(v)
    _bits_match(hi, wh, "split hi")
    _bits_match(lo, wl, "split lo")
    fin = torch.isfinite(hi)
    _split_ok(hi[fin].view(-1, 1), lo[fin].view(-1, 1))
    # 65 504 is exact; 65 519.996 keeps hi = 65 504 with lo = 16 (finite, but hi + lo = 65 520); 65 520 overflows
    i0 = sweep.size
    idx = {float(s): i0 + j for j, s in enumerate(special[:-1])}
    bits = lambda t, i: int(t[i].view(torch.int16)) & 0xFFFF
    assert (bits(hi, idx[65504.0]), bits(lo, idx[65504.0])) == (0x7BFF, 0x0000)
    j = idx[float(np.nextafter(np.float32(65520), np.float32(0)))]
    assert (bits(hi, j), bits(lo, j)) == (0x7BFF, 0x4C00)
    assert (bits(hi, idx[65520.0]), bits(lo, idx[65520.0])) == (0x7C00, 0xFC00)
    assert (bits(hi, idx[-65520.0]), bits(lo, idx[-65520.0])) == (0xFC00, 0x7C00)
    # join of the split: fp32(hi + lo) is exact, so it is the float64 sum rounded once
    with np.errstate(invalid="ignore"):
        _bits_match(_join_n(hi, lo), ref.join(wh, wl).astype(np.float32), "join of split")
    # join of every fp16 pattern as hi against random lo patterns (the float64 sum of two fp16 values is exact, so one
    # rounding to fp32 is what the fp32 add does), n not a multiple of 256
    ph = np.tile(np.arange(2 ** 16, dtype=np.uint16), 16)
    pl = rng.integers(0, 2 ** 16, ph.size).astype(np.uint16)
    ph, pl = np.r_[ph, ph[:5]], np.r_[pl, pl[:5]]
    with np.errstate(invalid="ignore"):
        want = ref.join(ph.view(np.float16), pl.view(np.float16)).astype(np.float32)
    got = _join_n(torch.from_numpy(ph.view(np.int16)).cuda().view(torch.float16),
                  torch.from_numpy(pl.view(np.int16)).cuda().view(torch.float16))
    _bits_match(got, want, "join of all patterns")
    # short lengths around the block of 256: nothing written past n
    for n in (1, 255, 257):
        h, l = _split_dev(torch.from_numpy(v[:n].copy()).cuda())
        _bits_match(h, wh[:n], f"split n={n}")
        with np.errstate(invalid="ignore"):
            _bits_match(_join_n(h, l), ref.join(wh[:n], wl[:n]).astype(np.float32), f"join n={n}")
    print(f"\nsplit / join: {v.size} and {ph.size} values bit-identical to the reference")
