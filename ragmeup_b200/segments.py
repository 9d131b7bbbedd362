"""Background segment writer shared by the stores that persist under a directory (``vectorstore``, ``pg_bm25``).

A store appends one segment file per change.  Segments are written by one background thread per store, in
submission order, so the device->host copies, the JSON tables and the file writes stay off the ingest loop.
``flush()`` waits for everything submitted so far and re-raises a writer error; it also runs at interpreter exit.
``RMU_STORE_SYNC=1`` writes inside ``submit`` instead.
"""
from __future__ import annotations

import atexit
import os
import queue
import threading
from typing import Any, Callable, Optional

import numpy as np


def atomic_savez(path: str, **arrays: Any) -> None:
    """``np.savez`` through a temporary name: a crash never leaves a half-written segment behind"""
    tmp = path + ".tmp.npz"
    np.savez(tmp, **arrays)
    os.replace(tmp, path)


class SegmentWriter:
    def __init__(self, write: Callable[..., None]):
        self._write = write
        self.sync = os.environ.get("RMU_STORE_SYNC", "0") == "1"
        self.thread: Optional[threading.Thread] = None
        self._queue: Optional["queue.Queue"] = None
        self._error: Optional[BaseException] = None

    def submit(self, *item: Any) -> None:
        """``write(*item)`` now (sync) or on the writer thread, after every item submitted before it"""
        if self.sync:
            self._write(*item)
            return
        if self.thread is None:
            self._queue = queue.Queue(maxsize=8)             # bounds the payloads kept alive for the writer
            self.thread = threading.Thread(target=self._loop, name="rmu-segment-writer", daemon=True)
            self.thread.start()
            atexit.register(self.flush)
        if self._error is not None:
            self.flush()
        self._queue.put(item)

    def _loop(self) -> None:
        while True:
            item = self._queue.get()
            try:
                if item is not None and self._error is None:
                    self._write(*item)
            except BaseException as e:                       # surfaced by the next submit / flush
                self._error = e
            finally:
                self._queue.task_done()
            if item is None:
                return

    def flush(self) -> None:
        """Wait until every segment submitted so far is on disk."""
        if self.thread is not None:
            self._queue.join()
        if self._error is not None:
            e, self._error = self._error, None
            raise RuntimeError(f"segment writer failed: {e!r}") from e
