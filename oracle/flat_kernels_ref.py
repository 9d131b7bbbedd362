"""Oracle: numpy restatements of the arithmetic the dense search kernels claim (``csrc/rmu_index.cu``,
``csrc/rmu_scan.cuh``).  TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

* ``tf32_trunc`` / ``tf32_rn``: an fp32 operand reduced to TF32 (10 explicit mantissa bits) by dropping the low 13 bits,
  or by rounding them to nearest even.  K1's ``wgmma ... tf32`` reads the fp32 corpus and queries as they lie in shared
  memory; which of the two the tensor core does is measured in ``tests/test_index_kernels_gpu.py``.
* ``exact_metric``: the fixed-order fp32 metric of ``exact_metric`` / ``exact_metric_quad`` (K2's re-score and K3): four
  interleaved ``fmaf`` chains over d = 4i + c, the D % 4 tail on chain 0, combined as (a0 + a1) + (a2 + a3); cosine
  divides by qnorm * sqrt(sum x^2) with the same four-chain sum of squares.
* ``query_norm``: ||q|| as K2 and K3 take it (256 threads with stride 256, warp xor butterfly, warp partials summed in
  order).
* ``row_sq_norm``: ``row_stats_kernel`` / ``set_rows_kernel``: one warp per row, lane l sums d = l, l + 32, ... with
  ``fmaf``, then an xor butterfly; lane 0's value is ||x||^2.
* ``coarse_key``: K1's epilogue on the TF32 accumulator: IP as is, cosine * 1/||x||, L2 + (-1/2 ||x||^2), nothing for
  cosine and L2 when the corpus counts as unit rows (max | ||x||^2 - 1 | < 1e-6).
* ``certificate``: ``kth_key``, ``eps`` and the second-pass threshold ``tau2`` exactly as ``select_rescore_kernel``
  writes them, in fp32.

``fmaf(a, b, c)`` is emulated as float32(float64(a) * float64(b) + float64(c)): the product of two fp32 values is exact
in float64, so the only departure from a single rounding is the rare double rounding of a sum that lands on an fp32
midpoint (at most one fp32 ulp).  nvcc may also contract ``a * b + c`` in the certificate into an fma; the emulation
rounds twice there.  Neither matters for the bounds the tests check.
"""
from __future__ import annotations

import numpy as np

METRICS = ("ip", "cosine", "l2")
EPS_REL = np.float32(2.2e-3)          # select_rescore_kernel's eps_rel (rmu_index.cu)
UNIT_DEV = np.float32(1e-6)           # max | ||x||^2 - 1 | below which rows count as unit rows
U32 = 2.0 ** -24                      # fp32 unit roundoff


def f32(a) -> np.ndarray:
    return np.asarray(a, dtype=np.float32)


def tf32_trunc(a) -> np.ndarray:
    """fp32 -> TF32 by dropping the low 13 mantissa bits (round toward zero)"""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    return (u & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_rn(a) -> np.ndarray:
    """fp32 -> TF32 rounded to nearest, ties to even (finite inputs)"""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = u + np.uint64(0x0FFF) + ((u >> np.uint64(13)) & np.uint64(1))
    return (u.astype(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def fmaf(a, b, c) -> np.ndarray:
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def exact_metric(q, x, metric: str, qnorm=None) -> np.ndarray:
    """[nq, D] x [N, D] -> fp32 [nq, N], the four-chain arithmetic of exact_metric.  ``qnorm`` [nq] (cosine) defaults to
    :func:`query_norm`."""
    q, x = f32(np.atleast_2d(q)), f32(np.atleast_2d(x))
    nq, D = q.shape
    N = x.shape[0]
    D4 = D & ~3
    a = [np.zeros((nq, N), np.float32) for _ in range(4)]
    n = [np.zeros((1, N), np.float32) for _ in range(4)]

    def step(c, d):
        if metric == "l2":
            e = (q[:, d:d + 1] - x[None, :, d]).astype(np.float32)
            a[c] = fmaf(e, e, a[c])
        else:
            a[c] = fmaf(q[:, d:d + 1], x[None, :, d], a[c])
            if metric == "cosine":
                n[c] = fmaf(x[None, :, d], x[None, :, d], n[c])

    for d0 in range(0, D4, 4):
        for c in range(4):
            step(c, d0 + c)
    for d in range(D4, D):
        step(0, d)
    s = (a[0] + a[1]) + (a[2] + a[3])
    if metric != "cosine":
        return s
    xn = np.sqrt((n[0] + n[1]) + (n[2] + n[3]))
    qn = query_norm(q) if qnorm is None else f32(qnorm)
    den = (qn[:, None] * xn).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(den > 0, s / np.where(den > 0, den, 1), 0).astype(np.float32)


def query_norm(q) -> np.ndarray:
    """[nq, D] -> fp32 [nq]: thread t < 256 sums d = t, t + 256, ... with fmaf; each warp reduces by xor butterfly; the
    eight warp partials are added in order (block_sum)"""
    q = f32(np.atleast_2d(q))
    nq, D = q.shape
    part = np.zeros((nq, 256), np.float32)
    for d0 in range(0, D, 256):
        w = min(256, D - d0)
        part[:, :w] = fmaf(q[:, d0:d0 + w], q[:, d0:d0 + w], part[:, :w])
    warps = _butterfly(part.reshape(nq, 8, 32))[..., 0]
    t = np.zeros(nq, np.float32)
    for w in range(8):
        t = (t + warps[:, w]).astype(np.float32)
    return np.sqrt(t)


def _butterfly(v) -> np.ndarray:
    """xor-shuffle reduction over the last axis (32 lanes): v[l] += v[l ^ o] for o = 16, 8, 4, 2, 1"""
    v = f32(v).copy()
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., lanes ^ o]).astype(np.float32)
    return v


def row_sq_norm(x) -> np.ndarray:
    """[N, D] -> fp32 [N] ||x||^2 as row_stats_kernel sums it (lane l: d = l, l + 32, ...; xor butterfly; lane 0)"""
    x = f32(np.atleast_2d(x))
    N, D = x.shape
    lane = np.zeros((N, 32), np.float32)
    for d0 in range(0, D, 32):
        w = min(32, D - d0)
        lane[:, :w] = fmaf(x[:, d0:d0 + w], x[:, d0:d0 + w], lane[:, :w])
    return _butterfly(lane)[:, 0]


def row_stats(x, metric: str):
    """-> (rscale, rbias, max ||x||, max | ||x||^2 - 1 |) as the index keeps them"""
    s = row_sq_norm(x)
    nrm = np.sqrt(s)
    with np.errstate(divide="ignore"):
        rscale = np.where(nrm > 0, np.float32(1) / np.where(nrm > 0, nrm, 1), 0).astype(np.float32)
    rbias = (np.float32(-0.5) * s).astype(np.float32)
    dev = np.abs((s - np.float32(1)).astype(np.float32))
    return rscale, rbias, np.float32(nrm.max()), np.float32(dev.max())


def unit_rows(max_dev) -> bool:
    return bool(np.float32(max_dev) < UNIT_DEV)


def tf32_dot(q, x, rounding: str = "trunc") -> np.ndarray:
    """float64 sum of the TF32 products (exact: two 11-bit significands fit fp32), no accumulation error"""
    t = tf32_trunc if rounding == "trunc" else tf32_rn
    return t(q).astype(np.float64) @ t(x).astype(np.float64).T


def coarse_key(acc, metric: str, rscale, rbias, unit: bool) -> np.ndarray:
    """K1's epilogue fmaf(acc, scale, bias) on fp32 accumulators [nq, N]"""
    acc = f32(acc)
    if metric == "cosine" and not unit:
        return fmaf(acc, f32(rscale)[None, :], np.float32(0))
    if metric == "l2" and not unit:
        return fmaf(acc, np.float32(1), f32(rbias)[None, :])
    return acc


def exact_key(v, metric: str, qnorm, unit: bool) -> np.ndarray:
    """an exact metric value in the units of the coarse key, float64: IP v; cosine v * ||q||;
    L2 (||q||^2 - dist) / 2 (+ 1/2 for unit rows, whose key leaves out -||x||^2 / 2)"""
    v = np.asarray(v, np.float64)
    qn = np.asarray(qnorm, np.float64).reshape(-1, 1)
    if metric == "ip":
        return v
    if metric == "cosine":
        return v * qn
    return 0.5 * (qn * qn - v) + (0.5 if unit else 0.0)


def certificate(metric: str, rk, qnorm, xmax, max_dev, eps_rel=EPS_REL):
    """(kth_key, eps, tau2) in fp32, as select_rescore_kernel computes them from the k-th exact rank value rk (the
    metric value, negated for L2), ||q||, max ||x|| and max | ||x||^2 - 1 |"""
    rk, qn, xmax, eps_rel = np.float32(rk), np.float32(qnorm), np.float32(xmax), np.float32(eps_rel)
    unit = unit_rows(max_dev) and metric != "ip"
    one, e6 = np.float32(1), np.float32(1e-6)
    if metric == "ip":
        kth, scale = rk, np.float32(qn * xmax)
    elif metric == "cosine":
        kth, scale = np.float32(rk * qn), qn
    else:
        kth = np.float32(np.float32(0.5) * np.float32(qn * qn + rk)) + (np.float32(0.5) if unit else np.float32(0))
        kth = np.float32(kth)
        scale = np.float32(qn * xmax)
    eps = np.float32(np.float32(eps_rel * scale) + np.float32(e6 * np.float32(one + abs(kth))))
    if unit:
        eps = np.float32(eps + np.float32(np.float32(4e-6) * np.float32(one + qn)))
    tau2 = np.float32(np.float32(kth - eps) - np.float32(e6 * np.float32(one + abs(kth))))
    return kth, eps, tau2
