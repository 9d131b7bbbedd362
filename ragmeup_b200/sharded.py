"""Row-sharded flat index across the GPUs of one box (SURVEY.md §8e).

The reference has no multi-device path; this is the GPU-native equivalent the north star asks for:
corpus rows are split contiguously over the ranks of a ``torch.distributed`` group (one process per
GPU), every rank scans only its shard, and ONE all-gather of the per-shard ``[Q, k]`` candidates
(fp32 scores + int64 global ids as one byte record per rank, <= 150 KB) over NCCL/NVLink feeds the on-device merge
(``rmu_topk_merge``).  Global ids are ``row + rank offset``, so results equal the unsharded search.
"""
from __future__ import annotations

from typing import Any, Callable, Optional, Tuple

import numpy as np


class ShardedFlatIndex:
    def __init__(self, local_index: Any, group: Any = None, merge_fn: Optional[Callable] = None):
        """``local_index``: a FlatIndex holding this rank's rows.  ``merge_fn(scores[R,Q,k], ids[R,Q,k],
        metric) -> (scores[Q,k], ids[Q,k])`` defaults to the CUDA merge kernel (tests inject another)."""
        import torch.distributed as dist
        self.dist = dist
        self.index = local_index
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        if merge_fn is None:
            from .index import topk_merge
            merge_fn = topk_merge
        self.merge_fn = merge_fn
        self._xkey, self._x = None, None
        self._preloaded = len(local_index)   # rows that were in the shard before the first add()
        self._batches = []          # sizes of the batches passed to add(), in order (identical on every rank)
        # what remove() took out, identical on every rank: per shard, the removed rows numbered among every row ever
        # added to that shard (sorted), and their positions in the order the batches were added (sorted, all shards)
        self._gone = [np.zeros(0, np.int64) for _ in range(self.world)]
        self._gone_pos = np.zeros(0, np.int64)
        self.offset = 0
        self.total = len(local_index)
        self._sizes = [len(local_index)]

    def sync_offsets(self) -> None:
        """Exchange shard sizes; rank r's ids start at sum(sizes[:r]).  Call after (re)loading shards."""
        import torch
        n = len(self.index)
        if self.world == 1:
            self._sizes, self.offset, self.total = [n], 0, n
            return
        dev = getattr(self.index, "device", torch.device("cpu"))
        mine = torch.tensor([n], dtype=torch.int64, device=dev)
        sizes = [torch.zeros_like(mine) for _ in range(self.world)]
        self.dist.all_gather(sizes, mine, group=self.group)
        self._sizes = [int(s.item()) for s in sizes]
        self.offset = sum(self._sizes[: self.rank])
        self.total = sum(self._sizes)

    # ------------------------------------------------------------------ sharded ingest (server/RAGHelper.py:423-434)
    def add(self, vectors) -> Tuple[int, int]:
        """The reference's ingest loop hands batches of 1000 documents to ``db.add_documents``; here EVERY rank is given
        the same batch [n, D] and keeps its block of it: rows [r*n//R, (r+1)*n//R).  Offsets are re-synchronised, so
        searches see the new rows at once.  Returns the (lo, hi) row range of the batch this rank kept."""
        n = int(vectors.shape[0])
        lo, hi = self.rank * n // self.world, (self.rank + 1) * n // self.world
        if hi > lo:
            self.index.add(vectors[lo:hi])
        self._batches.append(n)
        self._sizes = [s + ((r + 1) * n // self.world - r * n // self.world) for r, s in enumerate(self._sizes)] \
            if len(self._sizes) == self.world else None
        if self._sizes is None:
            self.sync_offsets()
        else:                                   # every rank can compute every shard size: no collective needed
            self.offset = sum(self._sizes[: self.rank])
            self.total = sum(self._sizes)
        return lo, hi

    def _layout(self):
        """per batch b and rank r: the first row of the batch the rank kept, where it starts in the rank's rows as if
        nothing were removed, and where the batch starts in the order the batches were added"""
        R = self.world
        nb = np.asarray(self._batches, np.int64)
        r = np.arange(R, dtype=np.int64)[:, None]
        first = r * nb // R                                                                        # [R, nb]
        local_start = np.concatenate([np.zeros((R, 1), np.int64), np.cumsum((r + 1) * nb // R - first, 1)], 1)
        batch_start = np.concatenate([[0], np.cumsum(nb)])
        return first, local_start, batch_start

    def _positions(self, r: int, local, layout):
        """current local rows of shard r -> their positions in the order the batches were added, removed rows counted"""
        first, local_start, batch_start = layout
        gone = self._gone[r]
        # the l-th surviving row is row l + #{removed rows before it} of everything the shard was given
        o = local + np.searchsorted(gone - np.arange(gone.size), local, side="right") if gone.size else local
        b = np.searchsorted(local_start[r], o, side="right") - 1
        return o, batch_start[b] + first[r, b] + (o - local_start[r, b])

    def remove(self, global_ids) -> int:
        """Every rank is handed the same merged ids (shard offset + local row, as :meth:`search` returns them; any order,
        duplicates allowed) and removes those that fall in its shard.  Each rank derives every shard's new size from the
        list, so offsets stay in step without a collective.  Raises ``ValueError`` on every rank, removing nothing, for
        an id outside ``[0, total)``.  Returns the number of rows this rank removed."""
        g = np.unique(np.asarray(global_ids.cpu() if hasattr(global_ids, "cpu") else global_ids, dtype=np.int64).reshape(-1))
        if self._sizes is None or len(self._sizes) != self.world:
            self.sync_offsets()
        if g.size and (g[0] < 0 or g[-1] >= self.total):
            raise ValueError(f"ids must lie in [0, {self.total})")
        starts = np.concatenate([[0], np.cumsum(self._sizes)])
        cuts = np.searchsorted(g, starts)
        mine = g[cuts[self.rank]:cuts[self.rank + 1]] - starts[self.rank]
        if mine.size:
            self.index.remove(mine)
        if not self._preloaded and g.size:
            layout = self._layout()
            found = [self._positions(r, g[cuts[r]:cuts[r + 1]] - starts[r], layout) for r in range(self.world)]
            for r, (o, _) in enumerate(found):
                self._gone[r] = np.union1d(self._gone[r], o)
            self._gone_pos = np.union1d(self._gone_pos, np.concatenate([pos for _, pos in found]))
        self._sizes = [s - int(cuts[r + 1] - cuts[r]) for r, s in enumerate(self._sizes)]
        self.offset = sum(self._sizes[: self.rank])
        self.total = sum(self._sizes)
        return int(mine.size)

    def to_insertion_order(self, ids):
        """merged global ids (shard offset + local row) -> position of the row among the surviving rows in the order the
        batches were added (what an unsharded store given the same adds and removes would call it); -1 stays -1.
        Only for shards filled through :meth:`add`."""
        if self._preloaded:
            raise ValueError("to_insertion_order needs shards that were filled through add() only")
        g = np.asarray(ids.cpu() if hasattr(ids, "cpu") else ids, dtype=np.int64)
        layout = self._layout()
        sizes = layout[1][:, -1] - np.array([gone.size for gone in self._gone], np.int64)
        offsets = np.concatenate([[0], np.cumsum(sizes)])
        out = np.full(g.shape, -1, np.int64)
        ok = g >= 0
        gk = g[ok]
        res = np.empty(gk.shape, np.int64)
        rk = np.searchsorted(offsets, gk, side="right") - 1
        for r in range(self.world):
            sel = rk == r
            if sel.any():
                _, pos = self._positions(r, gk[sel] - offsets[r], layout)
                res[sel] = pos - np.searchsorted(self._gone_pos, pos)      # removed rows before it do not count
        out[ok] = res
        return out

    def _exchange_buffers(self, Q: int, k: int, device):
        """One send record per rank: {scores fp32 [Q, k] | pad to 16 B | ids int64 [Q, k]} as raw bytes; the receive
        buffer holds the records of all ranks.  Views into both are created once per (Q, k)."""
        import torch
        key = (Q, k, str(device))
        if self._xkey != key:
            nb_s = Q * k * 4
            off_i = (nb_s + 15) // 16 * 16
            nb = off_i + Q * k * 8
            mine = torch.empty(nb, dtype=torch.uint8, device=device)
            allb = torch.empty((self.world, nb), dtype=torch.uint8, device=device)
            self._x = {
                "mine": mine, "all": allb.view(-1),       # concatenated form (the gloo backend only takes this one)
                "s": mine[:nb_s].view(torch.float32).view(Q, k), "i": mine[off_i:].view(torch.int64).view(Q, k),
                "gs": allb[:, :nb_s].view(torch.float32).view(self.world, Q, k),
                "gi": allb[:, off_i:].view(torch.int64).view(self.world, Q, k),
            }
            self._xkey = key
        return self._x

    def merge_gathered(self, s, i) -> Tuple[Any, Any]:
        """This rank's (scores [Q, k], global ids [Q, k]) -> ONE all-gather of the packed records -> merged top-k."""
        Q, k = s.shape
        x = self._exchange_buffers(Q, k, s.device)
        if s.data_ptr() != x["s"].data_ptr():
            x["s"].copy_(s)
            x["i"].copy_(i)
        self.dist.all_gather_into_tensor(x["all"], x["mine"], group=self.group)
        return self.merge_fn(x["gs"], x["gi"], self.index.metric)

    def search(self, queries, k: int) -> Tuple[Any, Any]:
        """Same queries on every rank -> the same merged (scores [Q,k], global ids [Q,k]) on every rank."""
        if self.world == 1:
            return self.index.search(queries, k, id_offset=self.offset)
        Q = queries.shape[0]
        dev = getattr(self.index, "device", queries.device)
        x = self._exchange_buffers(Q, k, dev)
        try:                                       # the CUDA index writes straight into the send record
            s, i = self.index.search(queries, k, id_offset=self.offset, out=(x["s"], x["i"]))
        except TypeError:                          # look-alikes without out= (CPU tests)
            s, i = self.index.search(queries, k, id_offset=self.offset)
        return self.merge_gathered(s, i)
