"""Continuous batching on the GPU decoder (rmu_decoder_session_*): every request that joins a session, whenever it
joins and whatever rows share its steps, gets bit for bit what rmu_decoder_generate returns for its prompt, settings
and seed, tokens and logits, on llama and qwen3, split and NF4, greedy and sampled.  Also: rows stopping by eos,
max_new_tokens and max_pos on different steps, 16 live rows and the busy answer, cache growth and cancellation with
live rows, other calls on the handle between steps, range errors that end only their own row, the per-row sampler
against one-row launches, DecoderAttention.generate from several threads, and two Llama-3.1-8B-shaped NF4 layers."""
from __future__ import annotations

import ctypes as C
import gc
import threading
from dataclasses import replace

import numpy as np
import pytest
import torch

import make_golden_generate as mg
from oracle import generation_ref as gref
from test_decode_batch_gpu import _batch, _handle, _prompts, _sampling, _single

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


class Tracker:
    """a DecodeSession with each request's tokens, logits and final status recorded by name"""

    def __init__(self, enc, V):
        from ragmeup_b200.decode_session import DecodeSession
        self.sess = DecodeSession(enc)
        self.V = V
        self.spec, self.slot, self.toks, self.logits, self.status = {}, {}, {}, {}, {}
        self.steps = 0

    def add(self, reqs):
        """reqs: [(name, ids, sampling, seed, max_new)]"""
        from ragmeup_b200.decode_session import Request
        lg = np.full((len(reqs), self.V), np.nan, np.float32)
        rows = self.sess.add([Request(ids, s, seed, mn) for _, ids, s, seed, mn in reqs], logits=lg)
        for i, ((name, ids, s, seed, mn), (slot, tok, st)) in enumerate(zip(reqs, rows)):
            self.spec[name] = (ids, s, seed, mn)
            self.toks[name], self.logits[name] = [], []
            self._record(name, slot, tok, st, lg[i])
        return rows

    def _record(self, name, slot, tok, st, lg):
        if st >= 0:
            self.toks[name].append(tok)
            self.logits[name].append(lg.copy())
        if st == _lib().GEN_LIVE:
            self.slot[slot] = name
        else:
            self.status[name] = st
            self.slot = {k: v for k, v in self.slot.items() if v != name}

    def step(self):
        lg = np.full((16, self.V), np.nan, np.float32)
        rows = self.sess.step(logits=lg)
        self.steps += 1
        for r, (slot, tok, st) in enumerate(rows):
            self._record(self.slot[slot], slot, tok, st, lg[r])
        return rows

    def live(self):
        return self.sess.info()[0]

    def run(self):
        while self.live():
            self.step()

    def check(self, enc, names=None):
        for name in names or list(self.spec):
            ids, s, seed, mn = self.spec[name]
            toks, lg = _single(enc, self.V, ids, s, seed, mn)
            assert self.toks[name] == toks, name
            got = np.stack(self.logits[name]) if self.logits[name] else np.zeros((0, self.V), np.float32)
            assert np.array_equal(got.view(np.int32), lg.view(np.int32)), name


SETTINGS = [_sampling(penalty=1.2), _sampling(True, 0.8, 40, 0.9, 1.3)]


@pytest.mark.parametrize("weights", ["split", "nf4"])
@pytest.mark.parametrize("kind", mg.KINDS)
def test_arrival_schedule_equals_solo_runs(kind, weights):
    """add A; 3 steps; add B and C (C a one-token prompt: the NF4 solo prefill); step until A stops; add D into A's
    freed region; run until every row stops"""
    cfg, w, lm, enc = _handle(kind, weights)
    V = cfg.vocab_size
    for i, s in enumerate(SETTINGS):
        p = _prompts(V, 4, 0, 3 + i, [30, 12, 1, 9])
        t = Tracker(enc, V)
        t.add([("A", p[0], s, 11, 8)])
        for _ in range(3):
            t.step()
        t.add([("B", p[1], s, 12, 14), ("C", p[2], s, 13, 10)])
        while "A" not in t.status:
            t.step()
        cap = t.sess.info()[1]
        t.add([("D", p[3], s, 14, 20)])                     # 9 + 20 <= 30 + 8: D fits A's freed region
        assert t.sess.info()[1] == cap
        t.run()
        assert t.status == {"A": 2, "B": 2, "C": 2, "D": 2}
        t.check(enc)


@pytest.mark.parametrize("weights", ["split", "nf4"])
def test_eos_and_max_pos_stops_on_different_steps(weights):
    cfg, w, lm, enc = _handle("llama", weights, max_pos=64)
    V = cfg.vocab_size
    p = _prompts(V, 4, 20, 9, [40, 30, 2, 38])               # totals 60, 50, 22, 58
    t = Tracker(enc, V)
    t.add([(str(b), p[b], _sampling(), 0, 12) for b in range(4)])
    t.run()
    t.check(enc)
    assert [len(t.toks[str(b)]) for b in range(4)] == [4, 12, 12, 6]
    assert [t.status[str(b)] for b in range(4)] == [3, 2, 2, 3]
    eos = (int(t.toks["1"][3]), int(t.toks["2"][6]))
    s = _sampling(eos=eos)
    t2 = Tracker(enc, V)
    t2.add([(str(b), p[b], s, 0, 12) for b in range(2)])
    t2.step()
    t2.add([(str(b), p[b], s, 0, 12) for b in range(2, 4)])
    t2.run()
    t2.check(enc)
    n = [len(t2.toks[str(b)]) for b in range(4)]
    assert len(set(n)) > 1 and 1 in t2.status.values()


def test_sixteen_rows_then_busy_changes_nothing():
    from ragmeup_b200.decode_session import SessionBusy
    cfg, w, lm, enc = _handle("qwen3", "nf4")
    V = cfg.vocab_size
    p = _prompts(V, 17, 5, 4)
    t = Tracker(enc, V)
    t.add([(str(b), p[b], SETTINGS[b % 2], b, 6) for b in range(10)])
    t.step()
    t.add([(str(b), p[b], SETTINGS[b % 2], b, 6) for b in range(10, 16)])
    before = t.sess.info()
    assert before[0] == 16
    with pytest.raises(SessionBusy):
        t.add([("16", p[16], SETTINGS[0], 16, 6)])
    assert t.sess.info() == before
    t.run()
    t.check(enc)


def test_mixed_settings_in_one_step():
    cfg, w, lm, enc = _handle("llama", "split")
    V = cfg.vocab_size
    p = _prompts(V, 6, 10, 8)
    settings = [_sampling(), _sampling(penalty=1.5), _sampling(True, 0.5, 10, 1.0), _sampling(True, 1.3, 200, 0.7, 1.1),
                _sampling(True, 1.0, 1), _sampling(True, 0.9, 50, 0.95, 0.8)]
    t = Tracker(enc, V)
    t.add([(str(b), p[b], settings[b], 2 ** 63 + 17 * b, 10) for b in range(6)])
    t.run()
    t.check(enc)


def test_cache_growth_with_live_rows():
    cfg, w, lm, enc = _handle("qwen3", "split")
    V = cfg.vocab_size
    p = _prompts(V, 3, 0, 2, [20, 50, 7])
    t = Tracker(enc, V)
    t.add([("A", p[0], SETTINGS[1], 1, 30)])
    assert t.sess.info() == (1, 50)
    t.step()
    t.step()
    t.add([("B", p[1], SETTINGS[1], 2, 30)])                 # no gap of 80 rows: the cache grows mid-reply
    assert t.sess.info() == (2, 130)
    t.step()
    t.add([("C", p[2], SETTINGS[0], 3, 30)])
    assert t.sess.info() == (3, 167)
    t.run()
    t.check(enc)


def test_cancel_frees_the_region_for_the_next_add():
    cfg, w, lm, enc = _handle("llama", "nf4")
    V = cfg.vocab_size
    p = _prompts(V, 4, 0, 6, [10, 25, 8, 30])
    t = Tracker(enc, V)
    rows = t.add([("A", p[0], SETTINGS[0], 1, 12), ("B", p[1], SETTINGS[1], 2, 20), ("C", p[2], SETTINGS[1], 3, 12)])
    t.step()
    t.step()
    cap = t.sess.info()[1]
    t.sess.cancel(rows[1][0])
    t.slot.pop(rows[1][0])
    del t.spec["B"]
    assert t.sess.info() == (2, cap)
    t.add([("D", p[3], SETTINGS[1], 4, 15)])                 # 45 rows: B's region
    assert t.sess.info() == (3, cap)
    t.run()
    t.check(enc)


def test_other_calls_between_steps():
    """span_mass, rmu_decoder_generate, rmu_decoder_generate_batch and prompt lookup on the same handle between steps:
    the session's rows are unaffected, and so are those calls' results"""
    L = _lib()
    cfg, w, lm, enc = _handle("llama", "split")
    V = cfg.vocab_size
    p = _prompts(V, 5, 4, 12, [40, 22, 3, 18, 30])
    spans = torch.tensor([[0, 10], [10, 30], [30, 44]], dtype=torch.int32, device="cuda")
    ids_d = torch.tensor(p[0], dtype=torch.int32, device="cuda")

    def span_mass():
        out = torch.empty((3, 3), dtype=torch.float64, device="cuda")
        L.check(L.lib().rmu_decoder_attention_spans(enc._h, ids_d.data_ptr(), len(p[0]), spans.data_ptr(), 3,
                                                    out.data_ptr(), L.stream_ptr()), "spans")
        return out.cpu().numpy()

    def lookup():
        out = np.zeros(12, np.int32)
        n = C.c_int32()
        s = SETTINGS[0]
        L.check(L.lib().rmu_decoder_generate_lookup(enc._h, np.ascontiguousarray(p[4], np.int32).ctypes.data, len(p[4]),
                                                    C.byref(s), 5, 12, 4, 2, out.ctypes.data, C.byref(n), None, None,
                                                    L.stream_ptr()), "lookup")
        return out[:n.value].tolist()

    want = (span_mass(), _single(enc, V, p[3], SETTINGS[1], 9, 10), _batch(enc, V, p[1:4], SETTINGS[1], [1, 2, 3], 6),
            lookup())
    t = Tracker(enc, V)
    t.add([("A", p[0], SETTINGS[1], 1, 16), ("B", p[2], SETTINGS[0], 2, 16)])
    for i in range(12):
        t.step()
        got = (span_mass, lambda: _single(enc, V, p[3], SETTINGS[1], 9, 10),
               lambda: _batch(enc, V, p[1:4], SETTINGS[1], [1, 2, 3], 6), lookup)[i % 4]()
        ref = want[i % 4]
        if i % 4 == 0:
            assert np.array_equal(got.view(np.int64), ref.view(np.int64))
        elif i % 4 == 1:
            assert got[0] == ref[0] and np.array_equal(got[1].view(np.int32), ref[1].view(np.int32))
        elif i % 4 == 2:
            assert got[0] == 0 and np.array_equal(got[1], ref[1]) and np.array_equal(got[3].view(np.int32),
                                                                                    ref[3].view(np.int32))
        else:
            assert got == ref
    t.run()
    t.check(enc)


def test_range_error_on_every_request():
    cfg, w, lm, enc = _handle("llama", cfg_w_lm=mg.model("llama", scale=3000.0))
    V = cfg.vocab_size
    t = Tracker(enc, V)
    rows = t.add([("A", list(range(1, 30)), SETTINGS[0], 0, 4), ("B", list(range(1, 20)), SETTINGS[1], 0, 4)])
    assert [r[0] for r in rows] == [-1, -1] and [r[2] for r in rows] == [-4, -4]
    assert t.sess.info()[0] == 0 and t.step() == []
    rows = t.add([("C", list(range(1, 30)), SETTINGS[0], 0, 4)])
    assert rows[0][2] == -4 and t.sess.info()[0] == 0


@pytest.mark.parametrize("weights", ["split", "nf4"])
def test_range_error_ends_only_its_own_row(weights):
    """token z's embedding is infinite, so feeding it leaves fp16's range; it is request R's third greedy token and
    never appears in the other rows, so R ends with RMU_ERR_RANGE at the step that feeds z (as its solo run fails)
    while the others in that step finish bit for bit"""
    cfg, w, lm = mg.model("llama")
    V = cfg.vocab_size
    p = _prompts(V, 4, 0, 21, [15, 9, 30, 4])
    _, _, _, enc = _handle("llama", weights, cfg_w_lm=(cfg, w, lm))
    s = SETTINGS[0]               # repetition penalty 1.2: a redo that saw the first pass's presence bits would differ
    clean = [_single(enc, V, q, s, 0, 10)[0] for q in p]
    del enc
    others = set(t for q in p[1:] for t in q) | set(t for c in clean[1:] for t in c)
    j = next(j for j in range(2, 9) if clean[0][j] not in clean[0][:j] + p[0] and clean[0][j] not in others)
    z = clean[0][j]
    w = dict(w)
    w["embed_tokens.weight"] = w["embed_tokens.weight"].copy()
    w["embed_tokens.weight"][z] = np.inf
    _, _, _, enc = _handle("llama", weights, cfg_w_lm=(cfg, w, lm))
    L = _lib()
    out, n = np.zeros(10, np.int32), C.c_int32()
    assert L.lib().rmu_decoder_generate(enc._h, np.ascontiguousarray(p[0], np.int32).ctypes.data, len(p[0]), C.byref(s),
                                        0, 10, out.ctypes.data, C.byref(n), None, L.stream_ptr()) == -4
    t = Tracker(enc, V)
    t.add([(str(b), p[b], s, 0, 10) for b in range(4)])
    t.run()
    assert t.status["0"] == -4 and t.toks["0"] == clean[0][:j + 1]
    assert t.sess.info()[0] == 0
    t.check(enc, ["1", "2", "3"])


@pytest.mark.parametrize("sampled", [False, True])
def test_sampler_session_rows_equal_one_row_launches(sampled):
    """rmu_debug_sample_session_rows: row r samples with sequence seq[r]'s bits, seed, step and settings, and equals
    rmu_debug_sample on that row at u = philox(seed, step): token, processed logits and bits"""
    L = _lib()
    V, nseq = 5000, 6
    seq_h = [4, 0, 2, 5, 3]                                  # a session has one row per live slot; slot 1 is idle
    B = len(seq_h)
    words = (V + 31) // 32
    g = torch.Generator(device="cuda").manual_seed(3 + int(sampled))
    logits = torch.randn(B, V, device="cuda", generator=g) * 3
    pres = torch.randint(0, 2 ** 31 - 1, (nseq, words), dtype=torch.int32, device="cuda", generator=g)
    seeds_h = [2 ** 63 + 5, 7, 123456789, 0, 42, 9]
    steps_h = [0, 3, 999, 17, 2 ** 40, 5]
    if sampled:
        settings = [_sampling(True, 0.7, 40, 0.9, 1.3), _sampling(True, 1.0, 1), _sampling(True, 1.5, 256, 0.5),
                    _sampling(True, 0.3, 5, 1.0, 0.7), _sampling(), _sampling(True, 1.0, 50, 1.0)]
    else:
        settings = [_sampling(), _sampling(penalty=1.3), _sampling(penalty=0.6), _sampling(penalty=2.0),
                    _sampling(penalty=1.01), _sampling()]
    s_arr = (L.SamplingC * nseq)(*settings)
    seq = torch.tensor(seq_h, dtype=torch.int32, device="cuda")
    seeds = torch.tensor(np.array(seeds_h, dtype=np.uint64).view(np.int64), device="cuda")
    steps = torch.tensor(np.array(steps_h, dtype=np.uint64).view(np.int64), device="cuda")
    lg, pr = logits.clone(), pres.clone()
    tok = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    L.check(L.lib().rmu_debug_sample_session_rows(lg.data_ptr(), V, B, pr.data_ptr(), seq.data_ptr(), seeds.data_ptr(),
                                                  steps.data_ptr(), nseq, C.cast(s_arr, C.c_void_p), tok.data_ptr(),
                                                  L.stream_ptr()), "sample_session_rows")
    torch.cuda.synchronize()
    for r, q in enumerate(seq_h):
        l1, p1 = logits[r].clone(), pres[q].clone()
        t1 = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        u = gref.philox_uniform(seeds_h[q], steps_h[q])
        s = settings[q]
        L.check(L.lib().rmu_debug_sample(l1.data_ptr(), V, p1.data_ptr(), C.byref(s), float(u), t1.data_ptr(),
                                         L.stream_ptr()), "sample")
        torch.cuda.synchronize()
        assert int(tok[r]) == int(t1[0]), r
        assert torch.equal(lg[r].view(torch.int32), l1.view(torch.int32)) and torch.equal(pr[q], p1), r


def test_decoder_attention_generate_from_threads(tmp_path):
    """DecoderAttention.generate from 4 threads equals 4 solo calls; a request that arrives while another is mid-reply
    is admitted before the first one finishes (the scheduler's log)"""
    from ragmeup_b200 import provenance
    mg.save_chat_snapshot(str(tmp_path))
    dec = provenance.DecoderAttention(str(tmp_path))
    V = dec.cfg.vocab_size
    p = _prompts(V, 4, 3, 31, [20, 5, 1, 12])
    kws = [dict(), dict(do_sample=True, temperature=0.7, top_k=30, top_p=0.9, repetition_penalty=1.1, seed=4),
           dict(repetition_penalty=1.3), dict(do_sample=True, seed=99)]
    solo = [dec.generate(p[i], 40, **kws[i]) for i in range(4)]
    sched = dec.scheduler()
    sched.log = []
    n_log = 0
    # the first request's third step waits until the other three callers are queued
    step, count, mid, go = sched.session.step, [0], threading.Event(), threading.Event()

    def gated(*a, **k):
        count[0] += 1
        if count[0] == 3:
            mid.set()
            go.wait(30)
        return step(*a, **k)

    sched.session.step = gated
    got = [None] * 4

    def run(i):
        got[i] = dec.generate(p[i], 40, **kws[i])

    threads = [threading.Thread(target=run, args=(i,)) for i in range(4)]
    threads[0].start()
    assert mid.wait(30)
    for th in threads[1:]:
        th.start()
    for _ in range(3000):
        if len(sched._queue) == 3:
            break
        threading.Event().wait(0.01)
    go.set()
    for th in threads:
        th.join(120)
    sched.session.step = step
    assert got == solo
    log = sched.log[n_log:]
    first = log[0][1][0]
    last_step_of_first = max(i for i, (kind, ids) in enumerate(log) if kind == "step" and first in ids)
    later_adds = [i for i, (kind, ids) in enumerate(log) if kind == "add" and first not in ids]
    assert later_adds and later_adds[0] < last_step_of_first


def test_llama_8b_shape_two_layers_nf4_staggered():
    """two layers of the Llama-3.1-8B shape on NF4, 8 rows arriving one every 4 steps: each equals its solo run"""
    from ragmeup_b200.weights import DECODER_PRESETS, synthetic_llama_weights
    cfg = replace(DECODER_PRESETS["llama-3.1-8b"], layers=2, vocab_size=2048, max_pos=4096)
    w = synthetic_llama_weights(cfg, seed=4)
    lm = (np.random.default_rng(4).standard_normal((cfg.vocab_size, cfg.hidden)) * 0.05).astype(np.float32)
    cfg, w, lm, enc = _handle("llama", "nf4", cfg_w_lm=(cfg, w, lm))
    del w
    V = cfg.vocab_size
    p = _prompts(V, 8, 300, 6, [200, 150, 1, 64, 65, 120, 30, 199])
    t = Tracker(enc, V)
    for b in range(8):
        t.add([(str(b), p[b], _sampling(True, 0.6, 50, 0.9), b, 12)])
        for _ in range(4):
            if t.live():
                t.step()
    t.run()
    t.check(enc)
