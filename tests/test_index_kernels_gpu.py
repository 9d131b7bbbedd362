"""GPU: the dense search kernels one at a time and at their edges.  K1 (``scan_rows_kernel``, TF32 wgmma scan) through
``rmu_debug_scan_tile`` against float64 sums of the TF32 operands; K2's certificate (``select_rescore_kernel``) on rows
built to sit inside the TF32 error; the second pass (``pool_prepare_kernel``, pool-mode K1, ``pool_rescore_kernel``) on
batches that mix flagged and certified queries; K3 (``exact_scan_kernel``); the upsert kernel; the shard merge.  The
references are oracle/flat_kernels_ref.py (pinned on the CPU by tests/test_flat_kernels_ref_cpu.py) and float64.

Error unit u = 2^-24.  Each bound's constant is derived next to it; the measured worst ratios are printed (-s) and
recorded in DESIGN.md section 2."""
import math

import numpy as np
import pytest
import torch

from oracle import flat_kernels_ref as kref
from oracle import flat_ref

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
TOL = 1e-3
SENT = -1234.5678
EPS = 2.0 ** -10                 # TF32 truncation step relative to the significand


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _modes():
    from ragmeup_b200.index import MODE_AUTO, MODE_EXACT, MODE_TENSOR_NOFALLBACK
    return MODE_AUTO, MODE_EXACT, MODE_TENSOR_NOFALLBACK


def _block_cap(D):
    """queries per K1 launch at dim D (scan_block_cap): the resident operand, ceil(D / 32) K blocks padded to whole stages
    of KD = 2 blocks of NQ x 128 bytes each, must fit 96 KB; 0 = D goes to K3"""
    kd = 2
    kb = ((D + 31) // 32 + kd - 1) // kd * kd
    cap = 64
    while cap >= 16 and kb * cap * 128 > 96 * 1024:
        cap //= 2
    return cap if cap >= 16 else 0


def _index(x, metric):
    from ragmeup_b200.index import FlatIndex
    ix = FlatIndex(x.shape[1], metric)
    ix.add(x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x)).cuda())
    return ix


def _same(a, b):
    """bit-identical (scores compared as bits: -0 vs 0 and NaN would show)"""
    if a.dtype == torch.float32:
        return torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


def _auto_equals_exact(ix, q, k, id_offset=0):
    """AUTO must return what MODE_EXACT (K3 alone) returns, bit for bit; -> (scores, ids, last_stats of AUTO)"""
    AUTO, EXACT, _ = _modes()
    s0, i0 = ix.search(q, k, id_offset=id_offset, mode=EXACT)
    s1, i1 = ix.search(q, k, id_offset=id_offset, mode=AUTO, want_stats=True)
    bad = (~((i0 == i1).all(1) & (s0.view(torch.int32) == s1.view(torch.int32)).all(1))).nonzero().flatten().tolist()
    assert not bad, f"AUTO differs from EXACT for queries {bad[:16]} (stats {ix.last_stats})"
    return s1, i1, ix.last_stats


def _values64(q, x, metric):
    """float64 metric values [nq, N] on the device (flat_ref.metric_values' definitions)"""
    q64, x64 = q.to(torch.float64), x.to(torch.float64)
    if metric == "ip":
        return q64 @ x64.T
    if metric == "cosine":
        den = q64.norm(dim=1)[:, None] * x64.norm(dim=1)[None, :]
        return torch.where(den > 0, (q64 @ x64.T) / torch.where(den > 0, den, 1), 0)
    return (q64 * q64).sum(1)[:, None] - 2 * q64 @ x64.T + (x64 * x64).sum(1)[None, :]


def _check_topk_fp64(s, i, q, x, k, metric, id_offset=0):
    """tests/test_index_gpu.py's check, with the float64 values taken on the device: ids identical to an exact search
    up to fp32 near-ties, judged in float64 — returned scores within TOL, returned order sorted, and no excluded row
    better than the k-th returned one, with a slack of a few fp32 ulps of the score magnitude."""
    v = _values64(q, x, metric).cpu().numpy()
    i = i.cpu().numpy() - id_offset
    s = s.cpu().numpy().astype(np.float64)
    rank = v if metric == "l2" else -v
    eps = 8 * np.finfo(np.float32).eps * max(1.0, float(np.abs(v).max()))
    for r in range(q.shape[0]):
        ids = i[r]
        assert (ids >= 0).all() and len(set(ids.tolist())) == len(ids)
        got = rank[r, ids]
        assert np.abs(s[r] - v[r, ids]).max() <= TOL * max(1.0, float(np.abs(v[r, ids]).max()) * 1e-2)
        assert (got[:-1] <= got[1:] + eps).all()
        rest = np.delete(rank[r], ids)
        assert rest.min() >= got[-1] - eps


# ------------------------------------------------------------------------------------------- K1 accumulators
# C_ACC: wgmma m64nNk8 tf32 multiplies TF32 operands exactly (two 11-bit significands fit fp32) and adds each k8 step
# to the fp32 accumulator once.  As E1 measured for fp16, that addition rounds toward zero, so the D / 8 step errors do
# not cancel; each is below one ulp of the running sum, at most 2 u S with S = sum_d |tq_d tx_d|.  So
# |acc - sum tq tx| <= c u (D / 8) S with c = 2.  That is the bound of one rounding toward zero per k8 step; that the
# hardware sums the 8 products of a step without further loss is an assumption about its alignment, confirmed by
# measurement (worst 1.97, at D = 4 on operands at the worst truncation) and not proved.  The test
# also reports the ratio against u sqrt(D / 8) S, the growth random-signed data would show with unbiased rounding: on
# the H100 that ratio climbs with D (13.7 at D = 1536) while the linear one stays near 1, so the error grows as D.
C_ACC = 2.0
DIMS = [4, 32, 36, 100, 384, 388, 768, 1024, 1536]


def _scan_tile(ix, q, nq_alloc):
    lib = _lib()
    out = torch.full((nq_alloc, 256), SENT, dtype=torch.float32, device="cuda")
    lib.check(lib.lib().rmu_debug_scan_tile(ix._h, q.data_ptr(), q.shape[0], out.data_ptr(), lib.stream_ptr()),
              "rmu_debug_scan_tile")
    torch.cuda.synchronize()
    return out


def _worst_truncation(a):
    """|a| with its low 13 mantissa bits all ones: truncation drops (2^13 - 1) 2^-23 of the significand, rounding to
    nearest goes up instead, and the two references part by ~2^-10 of every product"""
    u = np.abs(a).astype(np.float32).view(np.uint32) | np.uint32(0x1FFF)
    return u.view(np.float32)


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("kind", ["random", "worst"])
def test_scan_accumulators_match_tf32_float64(cuda, D, kind):
    rng = np.random.default_rng(D + (7 if kind == "worst" else 0))
    nq = _block_cap(D)
    N = 200 if D in (36, 1024) else 300                    # 200: tile 1 is ragged, rows 200..255 do not exist
    x = rng.standard_normal((N, D)).astype(np.float32)
    q = rng.standard_normal((nq, D)).astype(np.float32)
    if kind == "worst":
        x, q = _worst_truncation(x), _worst_truncation(q)
        x[1::2] *= -1                                      # mixed signs between rows, one sign inside a product sum
    q[0] = x[5]
    ix = _index(x, "ip")
    qd = torch.from_numpy(q).cuda()
    out = _scan_tile(ix, qd, nq + 3)
    assert (out[nq:] == SENT).all(), "the scan tile wrote rows of query slots past nq"
    rows = min(N, 256)
    if rows < 256:
        assert (out[:nq, rows:] == 0).all(), "rows past the corpus must accumulate TMA's zero fill"
    acc = out[:nq, :rows].double().cpu().numpy()
    xs = x[:rows]
    t_trunc = kref.tf32_dot(q, xs, "trunc")
    t_rn = kref.tf32_dot(q, xs, "rn")
    S_t = np.abs(kref.tf32_trunc(q)).astype(np.float64) @ np.abs(kref.tf32_trunc(xs)).astype(np.float64).T
    S = np.abs(q).astype(np.float64) @ np.abs(xs).astype(np.float64).T
    steps = -(-D // 8)
    err = np.abs(acc - t_trunc)
    lin = float((err / (U * steps * S_t)).max())
    sq = float((err / (U * math.sqrt(steps) * S_t)).max())
    rn = float((np.abs(acc - t_rn) / (U * steps * S_t)).max())
    exact = np.asarray(q, np.float64) @ np.asarray(xs, np.float64).T
    rel = np.abs(acc - exact) / S
    qx = np.linalg.norm(q.astype(np.float64), axis=1)[:, None] * np.linalg.norm(xs.astype(np.float64), axis=1)[None, :]
    cert = float((np.abs(acc - exact) / (float(kref.EPS_REL) * qx)).max())
    print(f"\nK1 D={D} {kind}: |acc - trunc ref| / (u (D/8) S) = {lin:.3g}, / (u sqrt(D/8) S) = {sq:.3g}; "
          f"vs round-to-nearest ref {rn:.3g}; |acc - q.x| / S = {rel.max():.3g} (2^-9 = {2 ** -9:.3g}); "
          f"/ (eps_rel |q||x|) = {cert:.3g}")
    assert lin <= C_ACC, f"K1 accumulators off the truncated-TF32 sum by {lin:.3g} u (D/8) S"
    if kind == "worst":
        # truncation, not rounding: the round-to-nearest reference is off by up to ~2^-9 S, ~2^15 / (D / 8) in this
        # unit (126 at D = 1536 on the H100)
        assert rn > 25 * C_ACC
    assert (rel <= 2.0 ** -9 + C_ACC * U * steps).all()         # the two-operand truncation bound eps_rel rests on
    assert cert < 1.0


def test_scan_tile_refuses_shapes_the_scan_does_not_take(cuda):
    lib = _lib()
    out = torch.zeros((64, 256), device="cuda")
    q = torch.zeros((64, 1540), device="cuda")
    for D, nq in ((1540, 1), (50, 1), (388, 33), (768, 33), (1536, 17), (384, 65)):
        ix = _index(np.ones((300, D), np.float32), "ip")
        qq = q[:nq, :D].contiguous()
        assert lib.lib().rmu_debug_scan_tile(ix._h, qq.data_ptr(), nq, out.data_ptr(), lib.stream_ptr()) == -1, (D, nq)
    from ragmeup_b200.index import FlatIndex
    empty = FlatIndex(32, "ip")
    assert lib.lib().rmu_debug_scan_tile(empty._h, q.data_ptr(), 1, out.data_ptr(), lib.stream_ptr()) == -1
    ix = _index(np.ones((300, 1536), np.float32), "ip")                 # the largest block at the largest dim is taken
    ones = torch.ones((16, 1536), device="cuda")
    lib.check(lib.lib().rmu_debug_scan_tile(ix._h, ones.data_ptr(), 16, out.data_ptr(), lib.stream_ptr()))
    torch.cuda.synchronize()
    assert (out[:16] == 1536.0).all()


# ------------------------------------------------------------------------------------- certificate edge (K2)
# D = m = 32, q TF32-exact.  C is TF32-exact, so its coarse key is its exact key; B's entries are 1 + 2^-10 - 2^-23,
# which truncate to 1, so B's coarse key drops by ~m 2^-10 while its exact key stays above C's.  300 copies of C fill
# KEEP = 64 (k = 10), B is excluded, and so are 236 copies of C whose coarse key equals the k-th exact key: the
# certificate cannot pass, and the second pass collects the rows whose coarse key beats
#     tau2 = kth - eps - 1e-6 (1 + |kth|),   eps = eps_rel * scale + 1e-6 (1 + |kth|).
# B enters the pool, and the answer is exact, iff coarse(B) > tau2, i.e. iff eps_rel * scale + 2e-6 (1 + |kth|) exceeds
# the gap kth - coarse(B):
#   IP:     q = 1^m, C = (1 + 2^-10)^(m-1) 1, gap = (m - 1) 2^-10, scale = ||q|| max||x|| ~ m (1 + 2^-10)
#           -> eps_rel > ~(m - 1) / m 2^-10 = 9.46e-4;
#   cosine: q = 1^m, C = 1^(m-1) (1 + 2^-5) (cos = 1 - 1.5e-5), B's cosine is 1; keys are cos * ||q||, scale = ||q||;
#           coarse(B) = ||q|| (1 - ~2^-10), gap ~ ||q|| (2^-10 - 1.5e-5) -> eps_rel > ~9.6e-4;
#   L2:     q = 8 * 1^m (keys q.x - ||x||^2 / 2), C and B as for IP; B is closer (dist 32 (7 - 2^-10)^2 against
#           31 (7 - 2^-10)^2 + 49); gap = 31 * 8 * 2^-10 + ~2^-10, scale = ||q|| max||x|| ~ 8 m -> eps_rel > ~9.5e-4.
# The test derives each threshold with the fp32 emulation of oracle/flat_kernels_ref.py and requires it between 9e-4 and
# 2.2e-3.  Only one operand is truncated here: the two-operand half of the 2 * 2^-10 bound cannot be reached at the k-th
# row without raising that row's exact score too, so this probe is sharp to eps_rel ~ 2^-10, not to 2^-9.
#
# Where the copies of C lie matters.  K1's threshold exchange takes the minimum over four CTA groups (cta % 4, KEEP 64) of
# each group's published 16th-best key, and K2 gathers list entries strictly above it.  Copies spread over all four
# groups make that minimum C's own key, K2 gathers fewer than k rows, and the second pass then takes every row of the
# corpus (a full pool, or K3 past 16 384 rows) whatever eps is.  So the copies go to tiles that one CTA group scans.
EDGE_B_ROW, EDGE_NC = 9000, 300


def _one_group_rows(n, N, first_tile=8):
    """n rows in 128-row tiles that CTAs of exchange group 0 scan (grid = min(SMs, tiles), tile t on CTA t % grid)"""
    grid = min(torch.cuda.get_device_properties(0).multi_processor_count, -(-N // 128))
    tiles = [t for t in range(first_tile, N // 128) if (t % grid) % 4 == 0]
    rows = np.concatenate([np.arange(128 * t, 128 * t + 128) for t in tiles])[:n]
    assert len(rows) == n
    return rows


def _edge_corpus(metric, N=16384):
    m = 32
    rng = np.random.default_rng(5)
    x = (-0.5 * np.abs(rng.standard_normal((N, m)))).astype(np.float32)    # filler: far below on every metric
    c = np.ones(m, np.float32)
    if metric == "cosine":
        c[-1] = 1 + 2.0 ** -5
    else:
        c[:-1] = 1 + 2.0 ** -10
    crows = _one_group_rows(EDGE_NC, N)
    x[crows] = c
    x[EDGE_B_ROW] = np.float32(1 + 2.0 ** -10 - 2.0 ** -23)
    q = np.full((1, m), 8.0 if metric == "l2" else 1.0, np.float32)
    return x, q, crows


def _edge_threshold(metric, x, q, crows):
    """the eps_rel below which B misses the second pass's pool, from the fp32 emulation"""
    rscale, rbias, xmax, dev = kref.row_stats(x, metric)
    rows = [EDGE_B_ROW, crows[0]]
    coarse = kref.coarse_key(kref.tf32_dot(q, x[rows]).astype(np.float32), metric, rscale[rows], rbias[rows], False)[0]
    v = kref.exact_metric(q, x[rows], metric)[0]
    rk = -v if metric == "l2" else v
    assert rk[0] > rk[1], "B must beat C exactly"
    assert coarse[0] < coarse[1], "B's coarse key must fall below C's"
    qn = kref.query_norm(q)[0]
    lo, hi = 0.0, 1e-2
    for _ in range(60):
        mid = 0.5 * (lo + hi)
        _, _, tau2 = kref.certificate(metric, rk[1], qn, xmax, dev, eps_rel=mid)
        lo, hi = (lo, mid) if coarse[0] > tau2 else (mid, hi)
    return hi


@pytest.mark.parametrize("metric", ["ip", "cosine", "l2"])
def test_certificate_edge_rows_inside_the_tf32_error(cuda, metric):
    _, _, NOFALLBACK = _modes()
    x, q, crows = _edge_corpus(metric, N=20000)
    thr = _edge_threshold(metric, x, q, crows)
    print(f"\ncertificate edge {metric}: B reaches the pool for eps_rel > {thr:.4g}")
    assert 9e-4 < thr < float(kref.EPS_REL)
    ix = _index(x, metric)
    qd = torch.from_numpy(q).cuda()
    want = [EDGE_B_ROW] + crows[:9].tolist()
    s, i, stats = _auto_equals_exact(ix, qd, 10)
    assert i[0].tolist() == want
    assert stats == (1, 1, 0)                     # flagged, answered by a pool of ~301 rows (not all 20 000: K3)
    # the first pass alone misses B: the construction does sit inside the TF32 error
    _, i1 = ix.search(qd, 10, mode=NOFALLBACK, want_stats=True)
    assert EDGE_B_ROW not in i1[0].tolist() and ix.last_stats[0] == 1
    _check_topk_fp64(s, i, qd, ix.data(), 10, metric)


# --------------------------------------------------------------------------------------------- end to end
def _corpus(kind, metric, N, D, g):
    x = torch.randn(N, D, device="cuda", generator=g)
    if kind == "unit":
        return torch.nn.functional.normalize(x, dim=1)
    if kind == "outlier":                           # one row 50x longer: eps scales with max ||x||
        x[77] *= 50.0
    elif kind == "zero-rows":                       # cosine on rows of spread norms, some all zero (score 0)
        x = x * torch.exp(torch.randn(N, 1, device="cuda", generator=g))
        x[[5, 900, N - 1]] = 0.0
    elif kind == "big-x":                           # ||x|| = 100, ||q|| = 1e-3: eps_rel's term is tiny, 1e-6 |kth| covers
        x = 100.0 * torch.nn.functional.normalize(x, dim=1)
    elif kind == "big-q":
        x = 0.01 * torch.nn.functional.normalize(x, dim=1)
    return x


def _queries(kind, nq, D, x, g):
    q = torch.nn.functional.normalize(torch.randn(nq, D, device="cuda", generator=g), dim=1)
    if kind == "big-x":
        return 1e-3 * q
    if kind == "big-q":
        return 100.0 * q
    q[0] = x[min(123, x.shape[0] - 1)]              # an exact hit
    if kind == "zero-q" and nq > 1:
        q[1] = 0.0                                  # IP / cosine: every row scores 0, the lowest rows win
    return q


# (metric, D, N, nq, k, kind, id_offset): K1 takes D % 4 == 0 up to 1536, N >= 16 384, k <= 128
E2E = [
    ("ip", 4, 16384, 17, 1, "unit", 0),             # one 32-column K block, mostly zero fill; NQ = 32
    ("cosine", 36, 16385, 33, 21, "randn", 0),      # D % 32 = 4; KEEP 64 at its edge (3k = 63)
    ("l2", 100, 16385, 65, 22, "randn", 0),         # KEEP 128 (3k = 66); two launches (64 + 1)
    ("ip", 388, 16384, 64, 42, "unit", 0),          # NQ = 32 at 388: two launches; 3k = 126
    ("cosine", 1024, 16385, 16, 43, "randn", 0),    # KEEP 256 (3k = 129); NQ = 16
    ("l2", 1536, 128 * 200 + 1, 17, 128, "randn", 0),   # one row in the last tile; k = 128
    ("ip", 1536, 16384, 129, 10, "unit", 0),        # nine NQ = 16 launches
    ("l2", 384, 16384, 32, 1, "unit", 0),           # unit-rows L2 key
    ("cosine", 384, 16384, 1, 128, "unit", 3_000_000_000),   # id_offset past 2^31 on the tensor path
    ("ip", 384, 20000, 8, 10, "outlier", 0),
    ("cosine", 384, 20000, 8, 10, "zero-rows", 0),
    ("ip", 384, 16384, 4, 10, "zero-q", 0),         # the zero query's pool is exactly 16 384 rows: pool cap
    ("cosine", 384, 16384, 4, 10, "zero-q", 0),
    ("l2", 384, 16384, 4, 10, "zero-q", 0),
    ("l2", 384, 16384, 8, 10, "big-x", 0),
    ("l2", 1536, 16384, 8, 10, "big-x", 0),
    ("l2", 384, 16384, 8, 10, "big-q", 0),
    # K3 only: D > 1536, N < 16 384, k > 128
    ("cosine", 1540, 16384, 5, 10, "randn", 0),
    ("l2", 384, 16383, 3, 10, "randn", 0),
    ("ip", 384, 16384, 4, 129, "unit", 0),
]


@pytest.mark.parametrize("metric,D,N,nq,k,kind,id_offset", E2E)
def test_search_matrix(cuda, metric, D, N, nq, k, kind, id_offset):
    g = torch.Generator(device="cuda").manual_seed(D * 7 + N + nq + k)
    x = _corpus(kind, metric, N, D, g)
    q = _queries(kind, nq, D, x, g)
    ix = _index(x, metric)
    s, i, stats = _auto_equals_exact(ix, q, k, id_offset)
    tensor = D % 4 == 0 and _block_cap(D) > 0 and N >= 16384 and k <= 128
    if tensor:
        cap = _block_cap(D)
        assert stats[1] == -(-nq // cap), stats                 # first-pass launches
        assert 0 <= stats[2] <= stats[0] <= nq
    else:
        assert stats == (nq, 0, nq)
    _check_topk_fp64(s, i, q, x, k, metric, id_offset)
    if kind == "zero-q" and metric != "l2":
        assert i[1].tolist() == list(range(k)) and (s[1] == 0).all()


def test_misaligned_query_view_uses_the_exact_scan(cuda):
    _, EXACT, _ = _modes()
    g = torch.Generator(device="cuda").manual_seed(11)
    D, nq = 384, 6
    x = torch.nn.functional.normalize(torch.randn(16384, D, device="cuda", generator=g), dim=1)
    q = torch.nn.functional.normalize(torch.randn(nq, D, device="cuda", generator=g), dim=1)
    buf = torch.empty(nq * D + 1, device="cuda")
    qm = buf[1:].view(nq, D)                                    # contiguous, 4 bytes past a 16-byte boundary
    qm.copy_(q)
    assert qm.data_ptr() % 16 == 4
    ix = _index(x, "ip")
    s, i = ix.search(qm, 10, want_stats=True)
    assert ix.last_stats == (nq, 0, nq)                          # TMA cannot load it: K3
    s0, i0 = ix.search(q, 10, mode=EXACT)
    assert _same(i, i0) and _same(s, s0)


# ---------------------------------------------------------------- threshold of the unit-rows shortcut (K1 / K2)
# Rows with max | ||x||^2 - 1 | < 1e-6 are scanned without the per-row L2 bias; K2 then adds 4e-6 (1 + ||q||) to eps.
# With ||q|| = 1e-3 the eps_rel term is ~2e-6, so eps ~ 7e-6 for unit rows, ~3e-6 otherwise.  R has ||R||^2 = 1 - dev
# and q.R = q.C - dev / 4: its key q.x - ||x||^2 / 2 beats the 300 copies of C by dev / 4, but the unit-row key q.x puts
# it dev / 4 below them.  Treated as unit rows (dev < 1e-6) that error is under 2.5e-7 and covered; dev = 5e-5 counted
# as unit rows would be off by 1.25e-5 > eps and R would miss the second pass.  Either way the 300 tied copies of C
# flag the query and the second pass answers it from a pool of about 301 rows; a scan that dropped the bias while the
# certificate kept it (or the reverse) would flag nothing, or fill the pool past its 16 384 rows with the 20 000.
R_ROW = 9000


def _unit_edge_corpus(dev, N=20000, D=64, qn=1e-3):
    """-> (x float32 [N, D] with R at R_ROW, q [1, D], R): random unit rows, 300 unit copies of C in one exchange group,
    R as described above"""
    rng = np.random.default_rng(int(dev * 1e9))
    x = rng.standard_normal((N, D))
    x /= np.linalg.norm(x, axis=1, keepdims=True)                 # random rows: q.x below ~0.6 qn
    crows = _one_group_rows(300, N)                                # see the certificate-edge test above
    x[crows] = 0.0
    x[crows, 0], x[crows, 1] = 0.9, math.sqrt(1 - 0.81)          # q.C = 0.9 qn, ||C|| = 1
    cr = 0.9 - dev / 4 / qn
    r = np.zeros(D)
    r[0], r[1] = cr, math.sqrt(1 - dev - cr * cr)                  # ||R||^2 = 1 - dev
    x[R_ROW] = r
    q = np.zeros((1, D), np.float32)
    q[0, 0] = qn
    return x.astype(np.float32), q, r.astype(np.float32)


@pytest.mark.parametrize("dev", [8e-7, 1.3e-6, 5e-5])
def test_unit_rows_threshold_edges(cuda, dev):
    x, q, _ = _unit_edge_corpus(dev)
    _, _, _, mdev = kref.row_stats(x, "l2")
    assert (mdev < 1e-6) == (dev < 1e-6) and abs(float(mdev) - dev) < 1.5e-7, float(mdev)
    ix = _index(x, "l2")
    qd = torch.from_numpy(q).cuda()
    s, i, stats = _auto_equals_exact(ix, qd, 10)
    assert stats == (1, 1, 0), stats
    assert i[0, 0].item() == R_ROW
    _check_topk_fp64(s, i, qd, ix.data(), 10, "l2")


def test_row_norms_cover_the_columns_past_the_last_warp_stride(cuda):
    """L2 at D = 36 with most of each row's energy in columns 32..35.  A row bias -||x||^2 / 2 that left those columns out
    would raise every coarse key (the answer would stay exact, through the second pass) and flag every query; with the
    whole row summed, norm-dominated keys 10th and 64th apart by far more than eps certify at once."""
    g = torch.Generator(device="cuda").manual_seed(36)
    D, N, nq = 36, 16384, 8
    x = torch.randn(N, D, device="cuda", generator=g)
    x[:, 32:] *= 3.0
    q = torch.randn(nq, D, device="cuda", generator=g)
    ix = _index(x, "l2")
    s, i, stats = _auto_equals_exact(ix, q, 10)
    assert stats == (0, 1, 0), stats
    _check_topk_fp64(s, i, q, x, 10, "l2")


# ----------------------------------------------------------------------------------------------- second pass
def _clustered(g, n_clusters, per, n_rand, D, noise=2e-4):
    centers = torch.nn.functional.normalize(torch.randn(n_clusters, D, device="cuda", generator=g), dim=1)
    xc = centers.repeat_interleave(per, 0)
    xc = torch.nn.functional.normalize(xc + noise * torch.randn(xc.shape, device="cuda", generator=g), dim=1)
    xr = torch.nn.functional.normalize(torch.randn(n_rand, D, device="cuda", generator=g), dim=1)
    return centers, torch.cat([xc, xr])


def _near(centers, g, noise=2e-4):
    return torch.nn.functional.normalize(centers + noise * torch.randn(centers.shape, device="cuda", generator=g), dim=1)


@pytest.mark.parametrize("metric", ["ip", "cosine"])
def test_second_pass_mixed_flags(cuda, metric):
    """300 queries, every third one inside a cluster of 150 near-duplicates (flagged), the others mostly certified: the
    compacted map of flagged queries must send each pool to its own query.  The second pass takes min(300, 256) = 256
    slots in four 64-query pool-mode launches (q_off 0, 64, 128, 192); with at most 192 queries flagged the last one
    finds no live slot and exits at once (nq_dev)"""
    g = torch.Generator(device="cuda").manual_seed(21)
    D, nq = 384, 300
    centers, x = _clustered(g, 100, 150, 5000, D)
    q = torch.nn.functional.normalize(torch.randn(nq, D, device="cuda", generator=g), dim=1)
    q[0::3] = _near(centers, g)
    ix = _index(x, metric)
    s, i, stats = _auto_equals_exact(ix, q, 10)
    # the cluster queries are flagged, and so are the random queries whose best rows are a whole cluster (142 on the
    # H100); stats[1] counts the first pass's launches, ceil(300 / 64)
    assert 100 <= stats[0] <= 192 and stats[1] == 5 and stats[2] == 0, stats
    _check_topk_fp64(s, i, q, x, 10, metric)


def test_second_pass_takes_256_queries_and_k3_the_rest(cuda):
    """300 queries all flagged: the pool answers the first 256, K3 the last 44"""
    g = torch.Generator(device="cuda").manual_seed(22)
    D = 384
    centers, x = _clustered(g, 100, 150, 5000, D)
    q = _near(centers.repeat(3, 1), g)
    ix = _index(x, "ip")
    s, i, stats = _auto_equals_exact(ix, q, 10)
    assert stats == (300, 5, 44), stats
    _check_topk_fp64(s, i, q, x, 10, "ip")


def test_second_pass_one_pool_overflows(cuda):
    """query 1 sits in 17 000 near-copies of one row (its pool overflows 16 384 rows: K3 answers it), its neighbours in
    clusters of 150 (their pools answer them)"""
    g = torch.Generator(device="cuda").manual_seed(23)
    D = 384
    centers, x = _clustered(g, 100, 150, 0, D)
    big = torch.nn.functional.normalize(torch.randn(1, D, device="cuda", generator=g), dim=1)
    xb = torch.nn.functional.normalize(big.repeat(17_000, 1) + 1e-4 * torch.randn(17_000, D, device="cuda", generator=g), dim=1)
    x = torch.cat([x, xb])
    q = torch.cat([_near(centers[:1], g), _near(big, g), _near(centers[1:3], g)])
    ix = _index(x, "ip")
    s, i, stats = _auto_equals_exact(ix, q, 10)
    assert stats == (4, 1, 1), stats
    _check_topk_fp64(s, i, q, x, 10, "ip")


# ---------------------------------------------------------------------------------------------------- upsert
@pytest.mark.parametrize("case", ["unit-to-nonunit-cosine", "cosine-rscale", "l2-rbias", "ip-out-of-range"])
def test_set_rows_equals_a_fresh_index(cuda, case):
    """after set_rows the index must search bit-identically to one built from the updated matrix (AUTO and EXACT)"""
    metric = case.split("-")[-1] if case.startswith("unit") else case.split("-")[0]
    g = torch.Generator(device="cuda").manual_seed(len(case))
    D, N = 128, 16384
    x = torch.nn.functional.normalize(torch.randn(N, D, device="cuda", generator=g), dim=1)
    if not case.startswith("unit"):
        x = x * (1.0 + 2.0 * torch.rand(N, 1, device="cuda", generator=g))       # norms in [1, 3]
    q = torch.nn.functional.normalize(torch.randn(8, D, device="cuda", generator=g), dim=1)
    rows = torch.tensor([123, 4567], device="cuda")
    if case.startswith("unit"):
        # ||x|| = 0.1: the shortcut must turn off.  Left on, the scan would take q.x = 0.1 cos for the cosine key, far
        # below the random rows' best cosines (~0.3), and both rows (cosine 1) would go missing
        new = torch.stack([0.1 * q[0], 0.1 * q[1]])
    elif case == "cosine-rscale":
        x[rows] = 3.0 * torch.nn.functional.normalize(x[rows], dim=1)
        new = torch.stack([0.01 * q[0], 0.02 * q[1]])        # a stale 1/||x|| = 1/3 would sink them
    elif case == "l2-rbias":
        x[rows] = 3.0 * torch.nn.functional.normalize(x[rows], dim=1)
        new = torch.stack([q[0], q[1]])                      # a stale -||x||^2 / 2 = -4.5 would sink them
    else:
        rows = torch.tensor([N, -1, 7, N + 5], device="cuda")
        new = torch.stack([q[0], q[1], 2.0 * q[2], q[3]])
    ix = _index(x, metric)
    ix.set_rows(rows, new)
    upd = x.clone()
    ok = (rows >= 0) & (rows < N)
    upd[rows[ok]] = new[ok]
    assert len(ix) == N and torch.equal(ix.data(), upd)
    s1, i1 = _same_as_fresh(ix, upd, metric, q)
    _check_topk_fp64(s1, i1, q, upd, 10, metric)
    if case != "ip-out-of-range":
        assert i1[0, 0].item() == 123 and i1[1, 0].item() == 4567


def _same_as_fresh(ix, upd, metric, q, k=10, same_stats=False):
    """AUTO and EXACT on the upserted index equal, bit for bit, those of an index built from the updated matrix, and with
    `same_stats` with the same flag counts (not in general: an overwritten row leaves the running maxima where they were,
    which may flag more); -> the AUTO result"""
    AUTO, EXACT, _ = _modes()
    fresh = _index(upd, metric)
    for mode in (EXACT, AUTO):
        s0, i0 = fresh.search(q, k, mode=mode, want_stats=True)
        s1, i1 = ix.search(q, k, mode=mode, want_stats=True)
        assert _same(i0, i1) and _same(s0, s1), mode
        assert not same_stats or ix.last_stats == fresh.last_stats, (mode, ix.last_stats, fresh.last_stats)
    return s1, i1


def test_set_rows_refreshes_the_unit_rows_deviation(cuda):
    """the threshold-edge corpus at dev = 5e-5, built unit (R a random unit row), then R written by set_rows: max
    | ||x||^2 - 1 | must rise with it.  Left at its unit value, the scan would drop the L2 bias, R's key would fall 1.25e-5
    (> eps ~ 7e-6) below the copies of C and R would miss the second pass"""
    x, q, r = _unit_edge_corpus(5e-5)
    x0 = x.copy()
    rng = np.random.default_rng(9)
    v = rng.standard_normal(x.shape[1])
    x0[R_ROW] = (v / np.linalg.norm(v)).astype(np.float32)
    assert kref.row_stats(x0, "l2")[3] < 1e-6
    ix = _index(x0, "l2")
    ix.set_rows([R_ROW], torch.from_numpy(r[None]).cuda())
    qd = torch.from_numpy(q).cuda()
    s, i = _same_as_fresh(ix, torch.from_numpy(x).cuda(), "l2", qd, same_stats=True)
    assert ix.last_stats == (1, 1, 0) and i[0, 0].item() == R_ROW
    _check_topk_fp64(s, i, qd, ix.data(), 10, "l2")


def test_set_rows_refreshes_max_norm(cuda):
    """IP: an upserted row B whose norm is 64x the corpus's must raise max ||x||, which scales eps.  D = 64, q = 1^64,
    300 copies of C = 0^32 1^32 in one exchange group (key 32), filler far below with norm < ||C|| = sqrt(32).
    B = (64 a)^16 (-64)^16 (63/64)^32 with a = 1 + 2^-10 - 2^-23: a truncates to 1, so B's coarse key is 31.5 while its
    exact one is 31.5 + 1024 (2^-10 - 2^-23) ~ 32.5.  The copies of C flag the query; the second pass keeps B only if
    tau2 = 32 - eps - ... < 31.5, i.e. eps > ~0.5.  With ||B|| ~ 362 eps = 2.2e-3 * 8 * 362 ~ 6.4; with the stale
    max ||x|| = sqrt(32), eps ~ 0.1 and B would go missing."""
    D, N = 64, 20000
    rng = np.random.default_rng(64)
    x0 = (-0.15 * np.abs(rng.standard_normal((N, D)))).astype(np.float32)
    crows = _one_group_rows(300, N)
    x0[crows] = 0.0
    x0[crows, 32:] = 1.0
    a = np.float32(1 + 2.0 ** -10 - 2.0 ** -23)
    b = np.concatenate([np.full(16, 64 * a), np.full(16, -64.0), np.full(32, 63 / 64)]).astype(np.float32)
    q = np.ones((1, D), np.float32)
    x = x0.copy()
    x[EDGE_B_ROW] = b
    # the derivation, in the kernels' fp32 arithmetic
    coarse_b = float(kref.tf32_dot(q, b[None])[0, 0])
    assert coarse_b == 31.5 and kref.exact_metric(q, b[None], "ip")[0, 0] > 32.0
    _, _, xmax0, dev0 = kref.row_stats(x0, "ip")
    _, _, xmax, dev = kref.row_stats(x, "ip")
    assert xmax0 == np.float32(math.sqrt(32))
    assert kref.certificate("ip", 32.0, 8.0, xmax0, dev0)[2] > coarse_b > kref.certificate("ip", 32.0, 8.0, xmax, dev)[2]
    ix = _index(x0, "ip")
    ix.set_rows([EDGE_B_ROW], torch.from_numpy(b[None]).cuda())
    qd = torch.from_numpy(q).cuda()
    s, i = _same_as_fresh(ix, torch.from_numpy(x).cuda(), "ip", qd, same_stats=True)
    assert ix.last_stats == (1, 1, 0)
    assert i[0].tolist() == [EDGE_B_ROW] + crows[:9].tolist()
    _check_topk_fp64(s, i, qd, ix.data(), 10, "ip")


# ------------------------------------------------------------------------------------------------ shard merge
def _shard_lists(rng, R, nq, k, metric, nvalid, tie_levels):
    """per-shard lists as a shard's search returns them: best first, equal scores in ascending id order, -1 padding;
    scores drawn from `tie_levels` values so that ties cross shards, ids handed out so that a tied id of a later
    shard is often lower than one of an earlier shard"""
    missing = np.inf if metric == "l2" else -np.inf
    S = np.full((R, nq, k), missing, np.float32)
    I = np.full((R, nq, k), -1, np.int64)
    for r in range(R):
        for b in range(nq):
            n = nvalid[r]
            v = rng.integers(0, tie_levels, n).astype(np.float32) / 8
            ids = (R - r) * 100_000 + rng.choice(100_000, n, replace=False)
            order = np.lexsort((ids, v if metric == "l2" else -v))
            S[r, b, :n], I[r, b, :n] = v[order], ids[order]
    return S, I


@pytest.mark.parametrize("metric", ["ip", "l2"])
@pytest.mark.parametrize("R,k,nvalid", [(3, 10, (4, 0, 7)), (4, 1024, (1024, 1024, 1000, 1024)),
                                        (8, 512, (512,) * 8), (2, 16, (16, 16))])
def test_shard_merge_matches_the_oracle(cuda, metric, R, k, nvalid):
    from ragmeup_b200.index import topk_merge
    rng = np.random.default_rng(R * k)
    S, I = _shard_lists(rng, R, 5, k, metric, nvalid, tie_levels=max(4, k // 8))
    ms, mi = topk_merge(torch.from_numpy(S).cuda(), torch.from_numpy(I).cuda(), metric)
    rs, ri = flat_ref.shard_merge(S, I, metric)
    assert np.array_equal(mi.cpu().numpy(), ri)
    assert np.array_equal(ms.cpu().numpy(), rs)
