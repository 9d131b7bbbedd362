"""FlatIndex — torch-tensor view of the C-ABI flat vector index (``rmu_index_*``).

The exact-brute-force store that stands behind ``self.db`` of the reference
(``server/RAGHelper.py:388-404`` ctor, ``:431``/``:525`` add, ``:497-499`` search).  Tensors at this
boundary are CUDA fp32 / int64; the arithmetic is in ``csrc/rmu_index.cu``.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np

from . import _lib

METRICS = {"ip": 0, "cosine": 1, "l2": 2}
MODE_AUTO, MODE_EXACT, MODE_TENSOR_NOFALLBACK = 0, 1, 2


class FlatIndex:
    def __init__(self, dim: int, metric: str = "l2", device: Optional[int] = None):
        torch = _lib.require_cuda()
        if metric not in METRICS:
            raise ValueError(f"metric must be one of {sorted(METRICS)}, got {metric!r}")
        self.torch = torch
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.dim = int(dim)
        self.metric = metric
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_index_create(self.dim, METRICS[metric], C.byref(self._h)), "rmu_index_create")
        self.last_stats = (0, 0, 0)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                _lib.lib().rmu_index_destroy(h)
            except Exception:
                pass
            self._h = C.c_void_p()

    def __len__(self) -> int:
        return int(_lib.lib().rmu_index_size(self._h))

    @property
    def largest_is_best(self) -> bool:
        return self.metric != "l2"

    def reserve(self, rows: int) -> None:
        with self.torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_index_reserve(self._h, int(rows)), "rmu_index_reserve")

    def clear(self) -> None:
        with self.torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_index_clear(self._h), "rmu_index_clear")

    def add(self, vectors) -> None:
        """Append rows.  ``vectors``: CUDA/CPU torch tensor or numpy array [n, dim] (fp32)."""
        torch = self.torch
        if isinstance(vectors, np.ndarray):
            v = np.ascontiguousarray(vectors, dtype=np.float32)
            if v.ndim != 2 or v.shape[1] != self.dim:
                raise ValueError(f"expected [n, {self.dim}] vectors, got {v.shape}")
            with torch.cuda.device(self.device):
                _lib.check(_lib.lib().rmu_index_add(self._h, v.ctypes.data, v.shape[0], 1, _lib.stream_ptr()),
                           "rmu_index_add")
                torch.cuda.current_stream().synchronize()   # pageable source must outlive the copy
            return
        v = vectors.detach()
        if v.dim() != 2 or v.shape[1] != self.dim:
            raise ValueError(f"expected [n, {self.dim}] vectors, got {tuple(v.shape)}")
        v = v.to(dtype=torch.float32).contiguous()
        with torch.cuda.device(self.device):
            if v.is_cuda:
                if v.device != self.device:
                    v = v.to(self.device)
                _lib.check(_lib.lib().rmu_index_add(self._h, v.data_ptr(), v.shape[0], 0, _lib.stream_ptr()),
                           "rmu_index_add")
                v.record_stream(torch.cuda.current_stream())
            else:
                _lib.check(_lib.lib().rmu_index_add(self._h, v.data_ptr(), v.shape[0], 1, _lib.stream_ptr()),
                           "rmu_index_add")
                torch.cuda.current_stream().synchronize()

    def set_rows(self, rows, vectors) -> None:
        """Overwrite existing rows in place: ``rows`` (ints / int64 tensor, local row numbers), ``vectors`` [n, dim]."""
        torch = self.torch
        r = torch.as_tensor(rows, dtype=torch.int64).to(self.device).contiguous().view(-1)
        v = torch.as_tensor(vectors) if isinstance(vectors, np.ndarray) else vectors.detach()
        v = v.to(device=self.device, dtype=torch.float32).contiguous()
        if v.dim() != 2 or v.shape[1] != self.dim or v.shape[0] != r.numel():
            raise ValueError(f"expected {r.numel()} x {self.dim} vectors, got {tuple(v.shape)}")
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_index_set_rows(self._h, r.data_ptr(), v.data_ptr(), r.numel(), _lib.stream_ptr()),
                       "rmu_index_set_rows")
            r.record_stream(torch.cuda.current_stream())
            v.record_stream(torch.cuda.current_stream())

    def remove(self, rows) -> None:
        """Delete rows (ints, numpy or a tensor of local row numbers; any order, duplicates allowed).  The survivors
        close up in place and keep their order, so row numbers above a removed row shift down.  Runs on the current
        stream; raises ``RmuError`` (index untouched) for a row outside ``[0, len)``."""
        if hasattr(rows, "detach"):
            rows = rows.detach().cpu().numpy()
        r = np.ascontiguousarray(np.asarray(rows, dtype=np.int64).reshape(-1))
        with self.torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_index_remove(self._h, r.ctypes.data if r.size else None, r.size, _lib.stream_ptr()),
                       "rmu_index_remove")

    def search(self, queries, k: int, id_offset: int = 0, mode: int = MODE_AUTO,
               want_stats: bool = False, out=None) -> Tuple["object", "object"]:
        """queries CUDA fp32 [nq, dim] -> (scores fp32 [nq, k], ids int64 [nq, k]) on the device.

        Scores are the metric values (inner product / cosine similarity / squared L2 distance),
        best first; missing results (k > len) have id -1.  ``out=(scores, ids)``: contiguous CUDA tensors
        of those shapes to write into (e.g. views of a collective's send buffer)."""
        torch = self.torch
        q = queries.detach().to(device=self.device, dtype=torch.float32).contiguous()
        if q.dim() != 2 or q.shape[1] != self.dim:
            raise ValueError(f"expected [nq, {self.dim}] queries, got {tuple(q.shape)}")
        nq = q.shape[0]
        if out is None:
            scores = torch.empty((nq, k), dtype=torch.float32, device=self.device)
            ids = torch.empty((nq, k), dtype=torch.int64, device=self.device)
        else:
            scores, ids = out
            if (tuple(scores.shape) != (nq, k) or tuple(ids.shape) != (nq, k) or scores.dtype != torch.float32 or
                    ids.dtype != torch.int64 or not scores.is_contiguous() or not ids.is_contiguous() or
                    scores.device != self.device or ids.device != self.device):
                raise ValueError("out= must be contiguous CUDA (fp32 [nq, k], int64 [nq, k]) on the index device")
        stats = (C.c_int32 * 4)() if want_stats else None
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_index_search(self._h, q.data_ptr(), nq, int(k), int(id_offset), int(mode),
                                                   scores.data_ptr(), ids.data_ptr(),
                                                   C.cast(stats, C.c_void_p) if want_stats else None,
                                                   _lib.stream_ptr()), "rmu_index_search")
        if want_stats:
            self.last_stats = (int(stats[0]), int(stats[1]), int(stats[2]))
        return scores, ids

    def search_host(self, queries: np.ndarray, k: int, id_offset: int = 0, mode: int = MODE_AUTO):
        """Host numpy in, host numpy out (H2D + D2H inside the C call)."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        nq = q.shape[0]
        scores = np.empty((nq, k), dtype=np.float32)
        ids = np.empty((nq, k), dtype=np.int64)
        with self.torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_index_search_host(self._h, q.ctypes.data, nq, int(k), int(id_offset), int(mode),
                                                        scores.ctypes.data, ids.ctypes.data, _lib.stream_ptr()),
                       "rmu_index_search_host")
        return scores, ids

    def gather(self, rows):
        """rows int64 [n] (local row numbers) -> CUDA fp32 [n, dim]."""
        torch = self.torch
        r = rows.detach().to(device=self.device, dtype=torch.int64).contiguous().view(-1)
        out = torch.empty((r.numel(), self.dim), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_index_gather(self._h, r.data_ptr(), r.numel(), out.data_ptr(), _lib.stream_ptr()),
                       "rmu_index_gather")
        return out

    def data(self):
        """Zero-copy CUDA view [len, dim] of the stored fp32 corpus (persistence, tests)."""
        torch = self.torch
        n = len(self)
        if n == 0:
            return torch.empty((0, self.dim), dtype=torch.float32, device=self.device)
        ptr = _lib.lib().rmu_index_data(self._h)
        from torch.utils import dlpack  # noqa: F401  (ensure torch fully initialised)
        # build a tensor over the raw pointer through the CUDA array interface
        class _Raw:
            pass
        raw = _Raw()
        raw.__cuda_array_interface__ = {"shape": (n, self.dim), "typestr": "<f4", "data": (int(ptr), False),
                                        "version": 2}
        return torch.as_tensor(raw, device=self.device)


def topk_merge(scores, ids, metric: str):
    """[R, nq, k] per-shard results -> merged [nq, k] (``rmu_topk_merge_strided``).  The rank dimension may be
    strided (views into the receive buffer of one all-gather); the [nq, k] block of each rank must be dense."""
    torch = _lib.require_cuda()
    R, nq, k = scores.shape

    def dense_blocks(t):
        return t if (R == 1 or t[0].is_contiguous()) and t.stride(0) >= nq * k else t.contiguous()
    s = dense_blocks(scores)
    i = dense_blocks(ids)
    out_s = torch.empty((nq, k), dtype=torch.float32, device=s.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=s.device)
    with torch.cuda.device(s.device):
        _lib.check(_lib.lib().rmu_topk_merge_strided(s.data_ptr(), i.data_ptr(), s.stride(0) if R > 1 else nq * k,
                                                     i.stride(0) if R > 1 else nq * k, R, nq, k, METRICS[metric],
                                                     out_s.data_ptr(), out_i.data_ptr(), _lib.stream_ptr()),
                   "rmu_topk_merge_strided")
    return out_s, out_i


def mmr_select(q, cand, n_cand, k: int, lambda_mult: float = 0.5):
    """q [nq, D], cand [nq, fetch_k, D], n_cand int32 [nq] -> int32 [nq, k] positions (-1 padded)."""
    torch = _lib.require_cuda()
    q = q.contiguous().float()
    cand = cand.contiguous().float()
    nq, fk, D = cand.shape
    out = torch.empty((nq, k), dtype=torch.int32, device=q.device)
    nc = None if n_cand is None else n_cand.to(device=q.device, dtype=torch.int32).contiguous()
    with torch.cuda.device(q.device):
        _lib.check(_lib.lib().rmu_mmr_select(q.data_ptr(), cand.data_ptr(), None if nc is None else nc.data_ptr(),
                                             nq, fk, D, int(k), float(lambda_mult), out.data_ptr(), _lib.stream_ptr()),
                   "rmu_mmr_select")
    return out
