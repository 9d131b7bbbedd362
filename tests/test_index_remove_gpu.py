"""GPU: FlatIndex.remove (rmu_index_remove) — the in-place, order-keeping compaction of the corpus.

The contract: after ``remove(rows)`` the index is indistinguishable from a fresh index built by adding the surviving
rows in their order.  Every case compares the two: size, the stored bytes, search scores and ids bit for bit in AUTO and
EXACT mode at k = 1, 10, 100, the search statistics, gather and MMR picks.

The compaction kernel moves chunks of kCompactChunk = 24576 floats (64 rows at D = 384), one chunk per CTA and one CTA
per SM in a round, so a round is 64 · (SM count) rows at D = 384; the boundary cases put run ends on both edges and one
row either side.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from ragmeup_b200 import _lib  # noqa: E402
from ragmeup_b200.index import MODE_AUTO, MODE_EXACT, FlatIndex, mmr_select  # noqa: E402

CHUNK_FLOATS = 24576        # kCompactChunk in csrc/rmu_index.cu


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda")


def _index(x, metric, batches=1):
    idx = FlatIndex(x.shape[1], metric)
    for part in np.array_split(np.arange(len(x)), batches):
        if part.size:
            idx.add(torch.from_numpy(x[part]).cuda())
    return idx


def _queries(x, rng, nq=9):
    q = rng.standard_normal((nq, x.shape[1])).astype(np.float32)
    if len(x):
        q[:3] = x[rng.integers(0, len(x), 3)]          # exact hits and their near-duplicates
    return torch.from_numpy(q).cuda()


def assert_same(idx, fresh, q):
    """idx (after remove) and fresh (built from the survivors) answer everything identically"""
    assert len(idx) == len(fresh)
    a, b = idx.data(), fresh.data()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    n = len(fresh)
    for mode in (MODE_AUTO, MODE_EXACT):
        for k in (1, 10, 100):
            s1, i1 = idx.search(q, k, mode=mode, want_stats=True)
            s2, i2 = fresh.search(q, k, mode=mode, want_stats=True)
            assert torch.equal(i1, i2), (mode, k)
            assert torch.equal(s1.view(torch.int32), s2.view(torch.int32)), (mode, k)
            assert idx.last_stats == fresh.last_stats, (mode, k)
    if n == 0:
        return
    _, ids = fresh.search(q, min(20, n))
    g1, g2 = idx.gather(ids.view(-1)), fresh.gather(ids.view(-1))
    assert torch.equal(g1.view(torch.int32), g2.view(torch.int32))
    fk = ids.shape[1]
    n_cand = torch.full((q.shape[0],), fk, dtype=torch.int32, device=q.device)
    m1 = mmr_select(q, g1.view(q.shape[0], fk, -1), n_cand, 4)
    m2 = mmr_select(q, g2.view(q.shape[0], fk, -1), n_cand, 4)
    assert torch.equal(m1, m2)


def run_case(x, rows, metric, rng, batches=1):
    idx = _index(x, metric, batches)
    idx.remove(rows)
    keep = np.setdiff1d(np.arange(len(x)), np.asarray(rows, dtype=np.int64))
    fresh = _index(x[keep], metric)
    assert_same(idx, fresh, _queries(x[keep], rng))
    return idx, keep


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


PATTERNS = ["nothing", "first", "last", "middle", "run_start", "run_middle", "run_end", "every_other", "random_1pct",
            "random_50pct"] + [f"{edge}_edge{d:+d}" for edge in ("chunk", "round") for d in (-1, 0, 1)]


def _pattern(name, n, D):
    rng = np.random.default_rng(n + D)
    if name == "nothing":
        return []
    if name in ("first", "last", "middle"):
        return [{"first": 0, "last": n - 1, "middle": n // 2}[name]]
    if name.startswith("run_"):
        lo = {"run_start": 0, "run_middle": n // 2 - 500, "run_end": n - 1000}[name]
        return list(range(lo, lo + 1000))                    # one document's chunks
    if name == "every_other":
        return list(range(0, n, 2))
    if name.startswith("random_"):
        return sorted(rng.choice(n, n // (100 if name == "random_1pct" else 2), replace=False).tolist())
    edge, d = name.split("_edge")
    chunk_rows = -(-CHUNK_FLOATS // D)
    L = chunk_rows if edge == "chunk" else chunk_rows * _sms()  # rows per chunk / per round (one CTA per SM)
    f = 1000
    L += int(d)
    assert f + 2 + L < n
    return [f, f + 1 + L]                          # the run between the two removed rows is L rows long


@pytest.mark.parametrize("pattern", PATTERNS)
def test_remove_patterns_l2_384(cuda, pattern):
    rng = np.random.default_rng(1)
    x = rng.standard_normal((50_000, 384)).astype(np.float32)
    run_case(x, _pattern(pattern, 50_000, 384), "l2", rng, batches=3)


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("D", [1, 3, 4, 36, 384, 388, 768, 1536, 2048])
def test_remove_shapes(cuda, D, metric):
    rng = np.random.default_rng(D)
    shift = 2 * -(-CHUNK_FLOATS // D) + 7                        # a shift longer than two chunks
    n = max(20_000 if D <= 768 else 17_000, 3000 + shift + 20_000)
    x = rng.standard_normal((n, D)).astype(np.float32)
    rows = set(rng.choice(n, n // 100, replace=False).tolist())
    rows |= set(range(3000, 3000 + shift))
    rows |= {0, n - 1}
    run_case(x, sorted(rows), metric, rng)


def test_remove_two_million_rows_384(cuda):
    rng = np.random.default_rng(5)
    n = 2_000_000
    x = rng.standard_normal((n, 384), dtype=np.float32)
    rows = set(rng.choice(n, n // 100, replace=False).tolist()) | set(range(700_000, 701_000))
    run_case(x, sorted(rows), "l2", rng)


def test_remove_all_then_add(cuda):
    rng = np.random.default_rng(2)
    x = rng.standard_normal((20_000, 64)).astype(np.float32)
    idx = _index(x, "ip")
    idx.remove(np.arange(len(x))[::-1])
    assert len(idx) == 0
    y = rng.standard_normal((17_000, 64)).astype(np.float32) * 0.5
    idx.add(torch.from_numpy(y).cuda())
    assert_same(idx, _index(y, "ip"), _queries(y, rng))


@pytest.mark.parametrize("metric", ["ip", "l2"])
def test_remove_largest_norm_row(cuda, metric):
    rng = np.random.default_rng(3)
    x = rng.standard_normal((20_000, 128)).astype(np.float32)
    x[777] *= 64.0                                   # drives max ||x|| and with it the certificate's eps
    run_case(x, [777], metric, rng)


def test_remove_the_only_non_unit_row_cosine(cuda):
    rng = np.random.default_rng(4)
    x = rng.standard_normal((20_000, 96)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x[123] *= 3.0                                    # the corpus leaves the unit-rows shortcut because of this row
    run_case(x, [123], "cosine", rng)


@pytest.mark.parametrize("metric", ["ip", "l2", "cosine"])
def test_remove_resets_maxima_raised_by_set_rows(cuda, metric):
    rng = np.random.default_rng(6)
    x = rng.standard_normal((20_000, 64)).astype(np.float32)
    idx = _index(x, metric)
    idx.set_rows([10], torch.from_numpy(x[10:11] * 100.0).cuda())   # raises the running maxima ...
    idx.set_rows([10], torch.from_numpy(x[10:11]).cuda())           # ... which stay raised after the row is restored
    idx.remove([5000])
    keep = np.setdiff1d(np.arange(len(x)), [5000])
    assert_same(idx, _index(x[keep], metric), _queries(x[keep], rng))


def test_interleaved_add_remove_set_rows(cuda):
    rng = np.random.default_rng(7)
    D = 48
    rows = [rng.standard_normal((9000, D)).astype(np.float32)]
    idx = _index(rows[0], "l2")
    ref = rows[0]
    idx.remove([0, 5, 8999, 4000])
    ref = np.delete(ref, [0, 5, 8999, 4000], axis=0)
    more = rng.standard_normal((12_000, D)).astype(np.float32)
    idx.add(torch.from_numpy(more).cuda())
    ref = np.concatenate([ref, more])
    upd = rng.standard_normal((3, D)).astype(np.float32)
    idx.set_rows([1, 9000, 20_000], torch.from_numpy(upd).cuda())
    ref[[1, 9000, 20_000]] = upd
    drop = sorted(set(rng.choice(len(ref), 2000, replace=False).tolist()) | set(range(8000, 9500)))
    idx.remove(drop)
    ref = np.delete(ref, drop, axis=0)
    assert_same(idx, _index(ref, "l2"), _queries(ref, rng))


def test_search_on_the_same_stream_sees_the_removal(cuda):
    rng = np.random.default_rng(8)
    x = rng.standard_normal((30_000, 128)).astype(np.float32)
    idx = _index(x, "ip")
    fresh = _index(x[1:], "ip")
    q = torch.from_numpy(x[:4].copy()).cuda()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        idx.remove([0])
        s1, i1 = idx.search(q, 10)                    # enqueued behind the compaction, no synchronise in between
    s.synchronize()
    s2, i2 = fresh.search(q, 10)
    assert torch.equal(i1, i2) and torch.equal(s1.view(torch.int32), s2.view(torch.int32))


def test_remove_refusals_leave_the_index_untouched(cuda):
    rng = np.random.default_rng(9)
    x = rng.standard_normal((5000, 20)).astype(np.float32)
    idx = _index(x, "l2")
    before = idx.data().clone()
    for bad in ([-1], [len(x)], [3, len(x) + 7]):
        with pytest.raises(_lib.RmuError):
            idx.remove(bad)
    stream = _lib.stream_ptr()
    assert _lib.lib().rmu_index_remove(idx._h, None, 3, stream) == -1
    arr = (C.c_int64 * 1)(0)
    assert _lib.lib().rmu_index_remove(idx._h, arr, -1, stream) == -1
    assert _lib.lib().rmu_index_remove(None, arr, 1, stream) == -1
    n0 = _lib.launch_count()
    idx.remove([])
    assert _lib.launch_count() == n0                 # nothing to remove: nothing launched
    assert len(idx) == len(x) and torch.equal(idx.data().view(torch.int32), before.view(torch.int32))
    assert_same(idx, _index(x, "l2"), _queries(x, rng))


def test_duplicates_and_order_do_not_matter(cuda):
    rng = np.random.default_rng(10)
    x = rng.standard_normal((20_000, 36)).astype(np.float32)
    rows = rng.choice(len(x), 300, replace=False)
    a = _index(x, "cosine")
    a.remove(np.sort(rows))
    b = _index(x, "cosine")
    b.remove(torch.from_numpy(np.concatenate([rows[::-1], rows[:50]])))
    assert_same(b, a, _queries(x, rng))
