"""Continuous batching without a GPU: the decode session's region placement (rmu_debug_kv_regions, host only), the
caller-driven scheduler (decode_session.Scheduler) over a fake session, and HuggingFacePipeline letting two threads
generate at once."""
from __future__ import annotations

import threading

import numpy as np
import pytest

from ragmeup_b200 import _lib
from ragmeup_b200.decode_session import Request, Scheduler, SessionBusy


# ------------------------------------------------------------------------------------------------ region placement
def _regions(ops):
    ops = np.asarray(ops, dtype=np.int32)
    out = np.zeros(2 * len(ops), dtype=np.int32)
    assert _lib.lib().rmu_debug_kv_regions(ops.ctypes.data, len(ops), out.ctypes.data) == 0
    return [tuple(r) for r in out.reshape(-1, 2).tolist()]


def test_regions_first_fit_merge_and_growth():
    got = _regions([10, 20, 5, -10, 8, 12, 0, 30, -30, -30])
    assert got == [
        (0, 10), (10, 30), (30, 35),     # each placed after the last, the cap growing to fit
        (0, 35),                         # free [10, 30)
        (10, 35), (18, 35),              # first fit into the freed gap, twice
        (0, 35),                         # free [0, 10)
        (35, 65),                        # no gap of 30: growth past the last used region; no region moves
        (0, 65), (-1, 65)]               # free [30, 35); a base that holds no region


def test_regions_merge_neighbouring_gaps():
    # [0, 4) [4, 12) [12, 20) used; freeing the first two leaves one gap of 12 rows
    got = _regions([4, 8, 8, 0, -4, 12, 1])
    assert got[-2] == (0, 20) and got[-1] == (20, 21)


def test_regions_refusals():
    assert _lib.lib().rmu_debug_kv_regions(None, 1, None) == -1


# ------------------------------------------------------------------------------------------------ the scheduler
class FakeSession:
    """each request emits its prompt's first id + 1, + 2, ... and stops after max_new_tokens; a prompt starting with
    a negative id fails at admission (as a refusal does), 999 fails at its second step (as a range error does)"""

    def __init__(self, rows=16):
        self.rows = rows
        self.live = {}                   # slot -> [request, n]
        self.calls = []
        self.busy = 0                    # the next `busy` adds answer busy
        self.fail = None                 # the next step raises this after running (None: no failure)
        self.release_on_failure = True   # a failed step releases its rows, as rmu_decoder_session_step does

    def add(self, reqs):
        self.calls.append(("add", [r.ids[0] for r in reqs]))
        if self.busy:
            self.busy -= 1
            raise SessionBusy("busy")
        if any(r.ids[0] < 0 for r in reqs):
            raise _lib.RmuError("rmu_decoder_session_add failed (rc=-1): token id out of range")
        if len(self.live) + len(reqs) > self.rows:
            raise SessionBusy("no free row")
        out = []
        for r in reqs:
            slot = min(set(range(self.rows)) - set(self.live))
            tok = r.ids[0] + 1
            if r.max_new_tokens == 1:
                out.append((-1, tok, _lib.GEN_MAX_NEW))
            else:
                self.live[slot] = [r, 1]
                out.append((slot, tok, _lib.GEN_LIVE))
        return out

    def step(self):
        self.calls.append(("step", sorted(self.live)))
        out = []
        for slot in sorted(self.live):
            r, n = self.live[slot]
            n += 1
            if r.ids[0] == 999 and n == 2:
                out.append((slot, 0, _lib.ERR_RANGE))
                del self.live[slot]
                continue
            self.live[slot][1] = n
            status = _lib.GEN_MAX_NEW if n == r.max_new_tokens else _lib.GEN_LIVE
            out.append((slot, r.ids[0] + n, status))
            if status != _lib.GEN_LIVE:
                del self.live[slot]
        if self.fail is not None:
            e, self.fail = self.fail, None
            if self.release_on_failure and isinstance(e, Exception):
                self.live.clear()
            raise e
        return out

    def live_slots(self):
        return sorted(self.live)

    def cancel(self, slot):
        self.calls.append(("cancel", slot))
        if slot not in self.live:
            raise _lib.RmuError(f"rmu_decoder_session_cancel failed (rc=-1): row {slot} is not live")
        del self.live[slot]


def _req(first, n):
    return Request([first, 7, 7], None, 0, n)


def test_one_caller_gets_its_tokens():
    sched = Scheduler(FakeSession())
    assert sched.run(_req(10, 4)) == [11, 12, 13, 14]
    assert sched.run(_req(20, 1)) == [21]


def _gate(fake):
    """make the fake's first step wait until `release` is set; `entered` is set when it starts waiting"""
    entered, release = threading.Event(), threading.Event()
    step = fake.step

    def gated():
        if not entered.is_set():
            entered.set()
            release.wait(10)
        return step()

    fake.step = gated
    return entered, release


def _thread(fn, *args):
    t = threading.Thread(target=fn, args=args)
    t.start()
    return t


def _queued(sched, n):
    for _ in range(1000):
        if len(sched._queue) >= n:
            return
        threading.Event().wait(0.01)
    raise AssertionError("requests were not queued")


def test_admission_only_at_step_boundaries():
    """requests that arrive while a step runs join at the next boundary, together, while the first reply is live"""
    fake = FakeSession()
    entered, release = _gate(fake)
    sched = Scheduler(fake)
    out = {}
    ta = _thread(lambda: out.setdefault("a", sched.run(_req(100, 6))))
    assert entered.wait(10)                       # A's driver is inside its first step
    tb = _thread(lambda: out.setdefault("b", sched.run(_req(200, 3))))
    tc = _thread(lambda: out.setdefault("c", sched.run(_req(300, 2))))
    _queued(sched, 2)
    release.set()
    for t in (ta, tb, tc):
        t.join(10)
    assert out == {"a": [101, 102, 103, 104, 105, 106], "b": [201, 202, 203], "c": [301, 302]}
    assert fake.calls[:4] == [("add", [100]), ("step", [0]), ("add", [200, 300]), ("step", [0, 1, 2])]


def test_driver_hands_off_when_its_reply_is_done():
    """the first caller drives; when its short reply ends, the waiting caller with a longer one takes over"""
    fake = FakeSession()
    entered, release = _gate(fake)
    sched = Scheduler(fake)
    drivers = []
    drive = sched._drive

    def logged(req):
        drivers.append(req.ids[0])
        drive(req)

    sched._drive = logged
    out = {}
    t1 = _thread(lambda: out.setdefault("short", sched.run(_req(10, 3))))
    assert entered.wait(10)
    t2 = _thread(lambda: out.setdefault("long", sched.run(_req(20, 8))))
    _queued(sched, 1)
    release.set()
    t1.join(10)
    t2.join(10)
    assert out == {"short": [11, 12, 13], "long": list(range(21, 29))}
    assert drivers == [10, 20]


def test_a_waiting_caller_cancels_its_row_on_an_exception():
    fake = FakeSession()
    sched = Scheduler(fake)
    a = sched.submit(_req(10, 50))
    b = sched.submit(_req(20, 3))
    with sched._cond:
        sched._admit()                            # both admitted, as a driver does at a boundary
    assert (a.slot, b.slot) == (0, 1)

    def interrupted(timeout=None):
        raise KeyboardInterrupt

    # B's caller is interrupted while another caller drives
    sched._driving = True
    wait, sched._cond.wait = sched._cond.wait, interrupted
    with pytest.raises(KeyboardInterrupt):
        sched.wait(b)
    sched._cond.wait = wait
    sched._driving = False
    assert ("cancel", 1) in fake.calls and 1 not in fake.live and b.done
    assert sched.wait(a) == list(range(11, 61))   # A is unaffected


def test_busy_keeps_the_request_queued():
    fake = FakeSession()
    sched = Scheduler(fake)
    a = sched.submit(_req(10, 5))
    with sched._cond:
        sched._admit()
    fake.busy = 2
    b = sched.submit(_req(20, 2))
    assert sched.wait(a) == [11, 12, 13, 14, 15]
    assert sched.wait(b) == [21, 22]
    assert [c for c in fake.calls if c[0] == "add"][:3] == [("add", [10]), ("add", [20]), ("add", [20])]


def test_an_error_reaches_only_its_own_caller():
    fake = FakeSession()
    sched = Scheduler(fake)
    good, bad, worse = sched.submit(_req(10, 4)), sched.submit(_req(-5, 4)), sched.submit(_req(999, 4))
    assert sched.wait(good) == [11, 12, 13, 14]
    with pytest.raises(_lib.RmuError, match="token id out of range"):
        sched.wait(bad)
    with pytest.raises(_lib.RmuError, match="fp16 range"):
        sched.wait(worse)
    assert worse.tokens == [1000] and not fake.live


@pytest.mark.parametrize("releases", [True, False])
def test_a_failed_step_ends_its_rows_and_the_next_request_completes(releases):
    """a step that fails ends every live request with its error; no row stays live in the session, whether the
    session released them itself or not, and a later request gets its whole reply"""
    fake = FakeSession()
    fake.release_on_failure = releases
    sched = Scheduler(fake)
    a, b = sched.submit(_req(10, 6)), sched.submit(_req(20, 6))
    with sched._cond:
        sched._admit()
    fake.fail = _lib.RmuError("rmu_decoder_session_step failed (rc=-2): out of memory")
    for r in (a, b):
        with pytest.raises(_lib.RmuError, match="out of memory"):
            sched.wait(r)
    assert not fake.live and not sched._live
    assert sched.run(_req(30, 4)) == [31, 32, 33, 34]


def test_an_interrupted_driver_leaves_consistent_replies():
    """a KeyboardInterrupt in the driving thread after a step ran: the driver's caller gets it, the other live request
    ends with an error instead of silently missing that step's token, no row stays live, and the next request
    completes"""
    fake = FakeSession()
    sched = Scheduler(fake)
    a, b = sched.submit(_req(10, 6)), sched.submit(_req(20, 6))
    with sched._cond:
        sched._admit()
    fake.fail = KeyboardInterrupt()
    with pytest.raises(KeyboardInterrupt):
        sched.wait(a)
    with pytest.raises(_lib.RmuError, match="interrupted"):
        sched.wait(b)
    assert b.tokens == [21] and not fake.live and not sched._live
    assert sched.run(_req(30, 3)) == [31, 32, 33]


def test_the_step_log_is_off_unless_asked_for():
    sched = Scheduler(FakeSession())
    sched.run(_req(10, 5))
    assert sched.log is None
    sched.log = []
    r = sched.run(_req(20, 3))
    assert r == [21, 22, 23] and [k for k, _ in sched.log] == ["add", "step", "step"]


def test_concurrent_first_lookups_build_one_decoder(monkeypatch):
    """two threads asking for the same decoder at once get one instance, built once"""
    from ragmeup_b200 import provenance
    built = []
    both_in = threading.Barrier(2, timeout=10)

    class SlowDecoder:
        def __init__(self, name, device=None, weights="split"):
            built.append(name)
            threading.Event().wait(0.3)                # an upload takes a while

    class FakeCuda:
        @staticmethod
        def current_device():
            return 0

    class FakeTorch:
        cuda = FakeCuda

    monkeypatch.setattr(provenance, "DecoderAttention", SlowDecoder)
    monkeypatch.setattr(provenance._lib, "require_cuda", lambda: FakeTorch)
    monkeypatch.setattr(provenance, "_DECODERS", {})
    got = [None, None]

    def lookup(i):
        both_in.wait()
        got[i] = provenance._decoder("synthetic:slow")

    threads = [_thread(lookup, i) for i in range(2)]
    for t in threads:
        t.join(10)
    assert built == ["synthetic:slow"] and got[0] is got[1] and got[0] is not None


# ------------------------------------------------------------------------------------------------ the pipeline
def test_pipeline_generates_from_two_threads_at_once(monkeypatch):
    """two invokes from two threads are inside the decoder's generate at the same time: the wrapper's lock covers the
    pipeline's pre- and post-processing only"""
    transformers = pytest.importorskip("transformers")
    import torch
    from ragmeup_b200 import llms

    class Tok:
        eos_token_id = 0

    class Pipe:
        _preprocess_params, _forward_params, _postprocess_params = {}, {}, {}
        generation_config = transformers.GenerationConfig(max_new_tokens=3, do_sample=False)

        def preprocess(self, prompt, **kw):
            return {"input_ids": torch.tensor([[len(prompt), 1]]), "prompt_text": prompt}

        def postprocess(self, out, **kw):
            return [{"generated_text": " ".join(str(int(t)) for t in out["generated_sequence"][0, 0])}]

    barrier = threading.Barrier(2, timeout=10)

    class Stub:
        def generate(self, ids, seed=0, **kw):
            barrier.wait()                        # passes only when both threads are here at once
            return [ids[0] + 1, ids[0] + 2, ids[0] + 3][:kw["max_new_tokens"]]

    stub = Stub()
    monkeypatch.setattr(llms._PipelineGenerator, "_decoder", lambda self: stub)
    llm = llms.HuggingFacePipeline(pipeline=Pipe())
    out = {}
    threads = [threading.Thread(target=lambda p=p: out.setdefault(p, llm.invoke(p))) for p in ("ab", "abcd")]
    for t in threads:
        t.start()
    for t in threads:
        t.join(20)
    assert not any(t.is_alive() for t in threads)
    assert out == {"ab": "2 1 3 4 5", "abcd": "4 1 5 6 7"}
    # batch() submits every prompt before it waits on any: the same barrier passes
    assert llm.batch(["ab", "abcd"]) == ["2 1 3 4 5", "4 1 5 6 7"]
