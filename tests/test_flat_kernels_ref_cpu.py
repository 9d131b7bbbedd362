"""CPU: pins oracle/flat_kernels_ref.py, the numpy restatement of the dense search kernels' arithmetic, and checks on
emulated data that the certificate's eps covers |exact key - coarse key| in every regime the index serves.

Error unit u = 2^-24.  A chain of n fmaf / additions is off by at most gamma_n * S, gamma_n = n u / (1 - n u), with S the
sum of the magnitudes of its terms (Higham, "Accuracy and Stability of Numerical Algorithms", 2nd ed., section 3.1)."""
import numpy as np
import pytest

from oracle import flat_kernels_ref as ref
from oracle import flat_ref

U = ref.U32


def _gamma(n):
    return n * U / (1 - n * U)


def test_tf32_truncation_and_rounding_match_bit_masks():
    rng = np.random.default_rng(0)
    a = (rng.standard_normal(10_000) * np.exp2(rng.integers(-30, 30, 10_000))).astype(np.float32)
    bits = a.view(np.uint32)
    assert (ref.tf32_trunc(a).view(np.uint32) == bits & np.uint32(0xFFFFE000)).all()
    rel = (a.astype(np.float64) - ref.tf32_trunc(a)) / a
    assert (rel >= 0).all() and (rel < 2.0 ** -10).all()                # toward zero, under 2^-10
    r = ref.tf32_rn(a).astype(np.float64)
    assert (np.abs(a - r) <= 2.0 ** -11 * np.abs(a)).all()               # nearest: half the truncation step
    assert (ref.tf32_rn(a).view(np.uint32) & np.uint32(0x1FFF) == 0).all()
    # the low 13 bits all ones: truncation loses almost 2^-10, rounding goes up
    b = np.float32(1 + 2.0 ** -10 - 2.0 ** -23)
    assert ref.tf32_trunc(b) == np.float32(1.0) and ref.tf32_rn(b) == np.float32(1 + 2.0 ** -10)
    assert ref.tf32_rn(np.float32(1 + 2.0 ** -11)) == np.float32(1.0)    # a tie goes to the even TF32 value
    assert ref.tf32_rn(np.float32(1 + 3 * 2.0 ** -11)) == np.float32(1 + 2.0 ** -9)
    assert ref.tf32_trunc(np.float32(-b)) == np.float32(-1.0)


@pytest.mark.parametrize("metric", ["ip", "cosine", "l2"])
@pytest.mark.parametrize("D", [1, 3, 4, 36, 101, 384])
def test_exact_metric_chains_match_float64(metric, D):
    rng = np.random.default_rng(D)
    q = rng.standard_normal((3, D)).astype(np.float32)
    x = rng.standard_normal((200, D)).astype(np.float32)
    x[7] = 0.0                                                          # cosine: a zero row scores 0
    got = ref.exact_metric(q, x, metric).astype(np.float64)
    want = flat_ref.metric_values(q, x, metric, dtype=np.float64)
    n = D // 4 + D % 4 + 2                                              # longest chain + the two combining additions
    if metric == "ip":
        S = np.abs(q).astype(np.float64) @ np.abs(x).astype(np.float64).T
        assert (np.abs(got - want) <= _gamma(n) * S).all()
    elif metric == "l2":
        S = want                                                        # every term is non-negative
        assert (np.abs(got - want) <= _gamma(n + 2) * S).all()          # + the rounding of q - x, squared
    else:
        qn = np.linalg.norm(q.astype(np.float64), axis=1)[:, None]
        xn = np.linalg.norm(x.astype(np.float64), axis=1)[None, :]
        with np.errstate(divide="ignore", invalid="ignore"):
            S = np.where(xn > 0, (np.abs(q).astype(np.float64) @ np.abs(x).astype(np.float64).T) / (qn * xn), 0)
        assert (np.abs(got - want) <= _gamma(n + 8) * (S + np.abs(want))).all()   # + the two norms, sqrt, divide
        assert (got[:, 7] == 0).all()
    # the four chains really are four: on data where the order matters, a single chain gives other bits
    if D >= 36 and metric == "ip":
        one = np.zeros((3, 200), np.float32)
        for d in range(D):
            one = ref.fmaf(q[:, d:d + 1], x[None, :, d], one)
        assert (one != got.astype(np.float32)).any()


def test_query_norm_and_row_sq_norm_match_float64():
    rng = np.random.default_rng(3)
    for D in (4, 31, 32, 33, 384, 1536):
        x = rng.standard_normal((50, D)).astype(np.float32)
        want = (x.astype(np.float64) ** 2).sum(1)
        s = ref.row_sq_norm(x).astype(np.float64)
        assert (np.abs(s - want) <= _gamma(-(-D // 32) + 5) * want).all()
        qn = ref.query_norm(x).astype(np.float64)
        assert (np.abs(qn - np.sqrt(want)) <= _gamma(-(-D // 256) + 9) * np.sqrt(want)).all()
    # lanes stride the row: the first 32 columns go to lanes 0..31, column 32 back to lane 0
    x = np.zeros((1, 64), np.float32)
    x[0, 0], x[0, 32], x[0, 1] = 2.0 ** 12, 1.0, 2.0 ** -12
    assert ref.row_sq_norm(x)[0] == np.float32(2.0 ** 24 + 1)          # 2^24 + 1 in lane 0: exact by fma
    assert ref.row_sq_norm(x[:, :32])[0] == np.float32(2.0 ** 24)


def test_certificate_formulas():
    kth, eps, tau2 = ref.certificate("ip", 0.8, 1.0, 1.0, 0.5)
    assert kth == np.float32(0.8)
    assert abs(float(eps) - (2.2e-3 + 1.8e-6)) < 1e-9
    assert abs(float(tau2) - (0.8 - 2.2e-3 - 3.6e-6)) < 1e-7
    kth, eps, _ = ref.certificate("cosine", 0.5, 2.0, 7.0, 0.5)        # cosine: scale ||q||, max ||x|| plays no part
    assert kth == np.float32(1.0) and abs(float(eps) - (4.4e-3 + 2e-6)) < 1e-9
    kth, eps, _ = ref.certificate("l2", -0.5, 1.0, 1.0, 1e-7)          # unit rows: + 1/2 and the 4e-6 (1 + ||q||) term
    assert kth == np.float32(0.75) and abs(float(eps) - (2.2e-3 + 1.75e-6 + 8e-6)) < 1e-9
    kth, eps, _ = ref.certificate("l2", -0.5, 1.0, 1.0, 1e-6)          # 1e-6 is not below the threshold
    assert kth == np.float32(0.25) and abs(float(eps) - (2.2e-3 + 1.25e-6)) < 1e-9
    _, e2, _ = ref.certificate("ip", 0.8, 1.0, 1.0, 0.5, eps_rel=9e-4)
    assert e2 < eps


# --------------------------------------------------------------------------------------- soundness on emulated data
def _regime(kind, D, rng):
    """-> (metric, q [4, D], x [N, D])"""
    n = 1500
    g = rng.standard_normal
    unit = lambda a: (a / np.linalg.norm(a, axis=1, keepdims=True)).astype(np.float32)  # noqa: E731
    if kind.startswith("unit-"):
        x = unit(g((n, D)))
        q = unit(g((4, D)))
        q[0] = x[3]
        return kind[5:], q, x
    if kind == "ip-outlier":
        x = g((n, D)).astype(np.float32)
        x[11] *= 40.0
        return "ip", g((4, D)).astype(np.float32), x
    if kind == "cosine-nonunit":
        x = (g((n, D)) * np.exp(g((n, 1)))).astype(np.float32)
        return "cosine", g((4, D)).astype(np.float32), x
    ratio = {"l2-x/q=1e-3": (0.1, 100.0), "l2-x/q=1": (1.0, 1.0), "l2-x/q=1e3": (100.0, 0.1),
             "l2-x/q=1e5": (100.0, 1e-3)}[kind]
    x = (ratio[0] * unit(g((n, D)))).astype(np.float32)
    q = (ratio[1] * unit(g((4, D)))).astype(np.float32)
    return "l2", q, x


REGIMES = ["unit-ip", "unit-cosine", "unit-l2", "ip-outlier", "cosine-nonunit", "l2-x/q=1e-3", "l2-x/q=1",
           "l2-x/q=1e3", "l2-x/q=1e5"]


def soundness_ratio(metric, q, x, rounding="trunc", eps_rel=ref.EPS_REL):
    """max over (query, row) of |exact key - coarse key| / eps, with eps evaluated at that row's exact key (the row that
    can break the certificate is one whose exact key reaches the k-th).  The TF32 sum is taken without accumulation
    error (the GPU test measures that part separately: it is below 2 u D / 8 of sum |q x|)."""
    rscale, rbias, xmax, dev = ref.row_stats(x, metric)
    unit = ref.unit_rows(dev) and metric != "ip"
    coarse = ref.coarse_key(ref.tf32_dot(q, x, rounding).astype(np.float32), metric, rscale, rbias, unit)
    qn = ref.query_norm(q)
    v = ref.exact_metric(q, x, metric, qn)
    ek = ref.exact_key(v, metric, qn, unit)
    worst = 0.0
    for i in range(q.shape[0]):
        rk = -v[i] if metric == "l2" else v[i]
        eps = np.array([float(ref.certificate(metric, r, qn[i], xmax, dev, eps_rel)[1]) for r in rk], np.float64)
        worst = max(worst, float((np.abs(ek[i] - coarse[i].astype(np.float64)) / eps).max()))
    return worst


@pytest.mark.parametrize("D", [384, 1536])
@pytest.mark.parametrize("kind", REGIMES)
def test_certificate_eps_covers_the_emulated_coarse_error(kind, D):
    metric, q, x = _regime(kind, D, np.random.default_rng(D + len(kind)))
    r = soundness_ratio(metric, q, x)
    print(f"\n{kind} D={D}: worst |exact key - coarse key| / eps = {r:.3g}")
    assert r < 1.0


def _worst_truncation(a):
    """|a| with the low 13 mantissa bits all ones: truncation drops almost 2^-10 of every operand, all one way"""
    return (np.abs(a).astype(np.float32).view(np.uint32) | np.uint32(0x1FFF)).view(np.float32)


def test_soundness_at_the_worst_truncation_and_with_a_too_small_eps_rel():
    """one-signed products of operands that truncation shrinks by (2^13 - 1) 2^-23 / significand, between 2^-11 and
    2^-10, each: the coarse key is low by up to 2^-9 sum |q x| = 2^-9 ||q|| ||x|| for parallel q and x.  eps_rel = 2.2e-3
    covers it; 2^-10 does not, so the check above can fail"""
    metric, q, x = _regime("unit-ip", 384, np.random.default_rng(1))
    q, x = _worst_truncation(q), _worst_truncation(x)
    q[0] = x[3]
    r = soundness_ratio(metric, q, x)
    print(f"\nworst truncation, IP: {r:.3g}")
    assert 0.5 < r < 1.0
    assert soundness_ratio(metric, q, x, eps_rel=2.0 ** -10) > 1.0
