"""Continuous batching on the GPU decoder: concurrent ``generate`` calls share one decode session.

``DecodeSession`` wraps ``rmu_gen_session`` (``include/ragmeup_b200.h``): requests join it between steps, each step
runs every live row at once, and a row leaves when it stops.  Each reply is bit for bit what ``rmu_decoder_generate``
returns for the same prompt, settings and seed, whatever rows share its steps.

``Scheduler`` drives a session from its callers' own threads; there is no background thread.  The first caller to
arrive drives: at each step boundary it admits the queued requests, then runs one step and hands out the tokens.  The
others wait.  A driver whose own reply is done hands the role to a waiting caller.  A caller interrupted while waiting
cancels its own row, and an error reaches only the caller whose request caused it.
"""
from __future__ import annotations

import ctypes as C
import itertools
import threading
from collections import deque
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _lib

RANGE_MESSAGE = ("an activation entering a GEMM or attention left the fp16 range of the split planes (|x| > 65504); "
                 "the decoder cannot compute this model's activations for this input")


class SessionBusy(Exception):
    """the session has no free row, or its KV cache cannot grow while rows are live: retry after a step"""


class Request:
    """one reply: the prompt ids, the sampler settings (``_lib.SamplingC``), the seed and max_new_tokens; ``tokens``
    fills as the steps run"""
    _ids = itertools.count()

    def __init__(self, ids: Sequence[int], sampling, seed: int, max_new_tokens: int, name: str = "decoder"):
        self.id = next(Request._ids)
        self.ids = [int(t) for t in ids]
        self.sampling = sampling
        self.seed = int(seed) & (2 ** 64 - 1)
        self.max_new_tokens = int(max_new_tokens)
        self.name = name
        self.tokens: List[int] = []
        self.slot: Optional[int] = None
        self.done = False
        self.error: Optional[BaseException] = None


Row = Tuple[int, int, int]          # (slot, token, status)


class DecodeSession:
    """one ``rmu_gen_session`` of a decoder encoder (``encoder.BertEncoder`` with an LM head attached); the encoder
    outlives the session because the session holds it"""

    def __init__(self, encoder):
        self.encoder = encoder
        self.vocab = int(encoder.cfg.vocab_size)
        self._h = C.c_void_p()
        _lib.check(_lib.lib().rmu_decoder_session_create(encoder._h, C.byref(self._h)), "rmu_decoder_session_create")

    def close(self) -> None:
        h, self._h = self._h, C.c_void_p()
        if h:
            _lib.lib().rmu_decoder_session_destroy(h)

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001 (interpreter shutdown)
            pass

    def _raise(self, rc: int, what: str):
        if rc == _lib.ERR_BUSY:
            msg = _lib.lib().rmu_last_error()
            raise SessionBusy(msg.decode() if msg else "busy")
        _lib.check(rc, what)

    def add(self, reqs: Sequence[Request], logits: Optional[np.ndarray] = None) -> List[Row]:
        """admit ``reqs`` -> (slot, first token, status) per request; slot -1 when it stopped or failed"""
        B = len(reqs)
        ids = np.ascontiguousarray([t for r in reqs for t in r.ids], dtype=np.int32)
        cu = np.ascontiguousarray(np.cumsum([0] + [len(r.ids) for r in reqs]), dtype=np.int32)
        s = (_lib.SamplingC * B)(*[r.sampling for r in reqs])
        seeds = np.ascontiguousarray([r.seed for r in reqs], dtype=np.uint64)
        max_new = np.ascontiguousarray([r.max_new_tokens for r in reqs], dtype=np.int32)
        slot, tok, status = (np.zeros(B, dtype=np.int32) for _ in range(3))
        rc = _lib.lib().rmu_decoder_session_add(self._h, ids.ctypes.data, cu.ctypes.data, B, C.cast(s, C.c_void_p),
                                                seeds.ctypes.data, max_new.ctypes.data, slot.ctypes.data,
                                                tok.ctypes.data, status.ctypes.data,
                                                None if logits is None else logits.ctypes.data, self._stream())
        self._raise(rc, "rmu_decoder_session_add")
        return list(zip(slot.tolist(), tok.tolist(), status.tolist()))

    def step(self, logits: Optional[np.ndarray] = None) -> List[Row]:
        """one decode step over every live row -> (slot, token, status) per row, in slot order"""
        slot, tok, status = (np.zeros(_lib.MAX_GENERATE_BATCH, dtype=np.int32) for _ in range(3))
        n = C.c_int32(0)
        rc = _lib.lib().rmu_decoder_session_step(self._h, slot.ctypes.data, tok.ctypes.data, status.ctypes.data,
                                                 C.byref(n), None if logits is None else logits.ctypes.data,
                                                 self._stream())
        self._raise(rc, "rmu_decoder_session_step")
        k = n.value
        return list(zip(slot[:k].tolist(), tok[:k].tolist(), status[:k].tolist()))

    def cancel(self, slot: int) -> None:
        _lib.check(_lib.lib().rmu_decoder_session_cancel(self._h, int(slot)), "rmu_decoder_session_cancel")

    def info(self) -> Tuple[int, int]:
        """(live rows, KV cache capacity in positions)"""
        live, cap = C.c_int32(0), C.c_int32(0)
        _lib.check(_lib.lib().rmu_decoder_session_info(self._h, C.byref(live), C.byref(cap), None),
                   "rmu_decoder_session_info")
        return live.value, cap.value

    def live_slots(self) -> List[int]:
        """the slots of the session's live rows"""
        live, cap, mask = C.c_int32(0), C.c_int32(0), C.c_uint32(0)
        _lib.check(_lib.lib().rmu_decoder_session_info(self._h, C.byref(live), C.byref(cap), C.byref(mask)),
                   "rmu_decoder_session_info")
        return [i for i in range(_lib.MAX_GENERATE_BATCH) if mask.value >> i & 1]

    def _stream(self) -> int:
        import torch
        return _lib.stream_ptr(torch.cuda.current_stream(self.encoder.device))


class Scheduler:
    """caller-driven continuous batching over a session with ``add`` / ``step`` / ``cancel`` / ``live_slots``
    (``DecodeSession``, or a fake in tests).  ``log``, when set to a list, records what each step boundary did:
    ("add", [request ids]) and ("step", [request ids]); it is off by default, since the scheduler lives as long as the
    process that serves its decoder."""

    def __init__(self, session, max_rows: int = _lib.MAX_GENERATE_BATCH):
        self.session = session
        self.max_rows = max_rows
        self.log: Optional[list] = None
        self._cond = threading.Condition()
        self._queue: deque = deque()
        self._live: dict = {}                 # slot -> Request
        self._driving = False

    def submit(self, req: Request) -> Request:
        """queue ``req``; it is admitted at the next step boundary"""
        with self._cond:
            self._queue.append(req)
            self._cond.notify_all()
        return req

    def wait(self, req: Request) -> List[int]:
        """drive or wait until ``req`` is done -> its tokens; its own error is raised here"""
        with self._cond:
            try:
                while not req.done:
                    if not self._driving:
                        self._driving = True
                        try:
                            self._drive(req)
                        finally:
                            self._driving = False
                            self._cond.notify_all()
                    else:
                        self._cond.wait()
            except BaseException:
                self._abandon(req)
                raise
        if req.error is not None:
            raise req.error
        return req.tokens

    def run(self, req: Request) -> List[int]:
        return self.wait(self.submit(req))

    # -------------------------------------------------------------------- with self._cond held
    def _finish(self, req: Request, error: Optional[BaseException] = None) -> None:
        req.done = True
        req.error = error
        if req.slot is not None:
            self._live.pop(req.slot, None)
            req.slot = None

    def _abandon(self, req: Request) -> None:
        """the caller of ``req`` stopped waiting: drop it from the queue or cancel its row"""
        if req.done:
            return
        if req in self._queue:
            self._queue.remove(req)
        elif req.slot is not None and self._live.get(req.slot) is req:
            self._cancel(req.slot)             # a step in flight may have stopped the row already
        self._finish(req, req.error)
        self._cond.notify_all()

    def _unlocked(self, fn, *args):
        self._cond.release()
        try:
            return fn(*args)
        finally:
            self._cond.acquire()

    def _apply(self, req: Request, slot: int, tok: int, status: int) -> None:
        if status < 0:
            msg = RANGE_MESSAGE if status == _lib.ERR_RANGE else f"status {status}"
            self._finish(req, _lib.RmuError(f"{req.name}: rmu_decoder_generate failed: {msg}"))
            return
        req.tokens.append(tok)
        if status == _lib.GEN_LIVE:
            req.slot = slot
            self._live[slot] = req
        else:
            self._finish(req)

    def _record(self, kind: str, ids: List[int]) -> None:
        if self.log is not None:
            self.log.append((kind, ids))

    def _cancel(self, slot: int) -> None:
        try:
            self.session.cancel(slot)
        except _lib.RmuError:
            pass                               # the row has stopped already

    def _reconcile(self) -> None:
        """cancel every row of the session that no request here owns, after a call that failed or was interrupted"""
        try:
            slots = self.session.live_slots()
        except Exception:  # noqa: BLE001 (the session is unusable; there is nothing to cancel)
            return
        for slot in slots:
            if slot not in self._live:
                self._cancel(slot)

    def _fail(self, reqs, error: BaseException) -> None:
        """end ``reqs`` with ``error`` and release whatever rows they held"""
        for r in list(reqs):
            if not r.done:
                self._finish(r, error)
        self._reconcile()
        self._cond.notify_all()

    @staticmethod
    def _interrupted(e: BaseException) -> _lib.RmuError:
        return _lib.RmuError(f"rmu_decoder_generate failed: the decode step was interrupted ({type(e).__name__})")

    def _admit(self, limit: int = _lib.MAX_GENERATE_BATCH) -> None:
        free = self.max_rows - len(self._live)
        batch = [self._queue.popleft() for _ in range(min(free, len(self._queue), limit))]
        if not batch:
            return
        try:
            rows = self._unlocked(self.session.add, batch)
        except SessionBusy:
            self._queue.extendleft(reversed(batch))
            if not self._live:
                raise
            return
        except Exception as e:  # noqa: BLE001
            if len(batch) == 1:
                self._fail(batch, e)
            else:
                # a refusal names one request: try each alone so that the error reaches only its own caller
                self._queue.extendleft(reversed(batch))
                self._admit(limit=1)
            return
        except BaseException as e:
            # interrupted after the add may have run: its requests end, and rows nobody owns are released
            self._fail(batch, self._interrupted(e))
            raise
        try:
            self._record("add", [r.id for r in batch])
            for r, (slot, tok, status) in zip(batch, rows):
                if r.done:                     # abandoned while the add ran
                    if status == _lib.GEN_LIVE:
                        self._cancel(slot)
                    continue
                self._apply(r, slot, tok, status)
        except BaseException as e:
            self._fail(batch, self._interrupted(e))
            raise
        self._cond.notify_all()

    def _step(self) -> None:
        try:
            rows = self._unlocked(self.session.step)
        except Exception as e:  # noqa: BLE001
            # a failed step leaves no row usable: every live request gets the error and no row stays live
            self._fail(self._live.values(), e)
            return
        except BaseException as e:
            self._fail(self._live.values(), self._interrupted(e))
            raise
        try:
            self._record("step", [self._live[s].id for s, _, _ in rows if s in self._live])
            for slot, tok, status in rows:
                r = self._live.get(slot)
                if r is not None:
                    self._apply(r, slot, tok, status)
        except BaseException as e:
            # a reply must not silently miss this step's token: the ones still live end with an error
            self._fail(self._live.values(), self._interrupted(e))
            raise
        self._cond.notify_all()

    def _drive(self, req: Request) -> None:
        """admit, step, hand out, until ``req`` is done"""
        while not req.done:
            if self._queue:
                try:
                    self._admit()
                except SessionBusy as e:
                    # busy with no live row: the request cannot be admitted
                    r = self._queue.popleft()
                    self._finish(r, _lib.RmuError(f"{r.name}: rmu_decoder_generate failed: {e}"))
                    self._cond.notify_all()
                if req.done:
                    break
            if self._live:
                self._step()
            elif not self._queue:
                break
