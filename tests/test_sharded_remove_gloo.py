"""CPU, world size 2 over gloo: ShardedFlatIndex.remove.  Every rank is handed the same merged ids and removes those in
its shard; offsets follow without a collective, and merged ids still map, through to_insertion_order, to the position
an unsharded index given the same adds and removes reports."""
import os

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


class RemovableShard:
    """FlatIndex look-alike over numpy with ``remove`` (the product index needs a GPU; the plumbing is under test)."""

    def __init__(self, dim, metric):
        self.x, self.metric, self.device = np.zeros((0, dim), np.float32), metric, torch.device("cpu")

    def __len__(self):
        return self.x.shape[0]

    def add(self, v):
        self.x = np.concatenate([self.x, np.asarray(v, np.float32)])

    def remove(self, rows):
        rows = np.asarray(rows, np.int64)
        assert rows.min() >= 0 and rows.max() < len(self.x)
        self.x = np.delete(self.x, rows, axis=0)

    def search(self, q, k, id_offset=0):
        from oracle import flat_ref
        s, i = flat_ref.flat_search(q.numpy(), self.x, k, self.metric, id_offset=id_offset)
        return torch.from_numpy(s), torch.from_numpy(i)


def oracle_merge(gs, gi, metric):
    from oracle import flat_ref
    s, i = flat_ref.shard_merge(gs.numpy(), gi.numpy(), metric)
    return torch.from_numpy(s), torch.from_numpy(i)


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle import flat_ref
        from ragmeup_b200.sharded import ShardedFlatIndex
        rng = np.random.default_rng(21)
        D = 16
        sh = ShardedFlatIndex(RemovableShard(D, "l2"), merge_fn=oracle_merge)
        sh.sync_offsets()
        # the test's own bookkeeping, independent of the code under test: every row ever added has a position in add
        # order and a vector; each shard holds the positions of its block of every batch, in row order
        vec = {}
        shard_pos = [[] for _ in range(world)]
        collectives = []
        real_all_gather = dist.all_gather
        dist.all_gather = lambda *a, **k: (collectives.append(1), real_all_gather(*a, **k))[1]
        ok = True
        added = 0
        for step, n in enumerate((37, 1000, 5, 400)):
            b = rng.standard_normal((n, D)).astype(np.float32)
            sh.add(b)
            for j in range(n):
                vec[added + j] = b[j]
            for r in range(world):
                shard_pos[r] += list(range(added + r * n // world, added + (r + 1) * n // world))
            added += n
            merged = [p for r in range(world) for p in shard_pos[r]]          # merged id -> position
            # merged ids to drop, as a search would return them: some from each shard, with duplicates, unsorted
            g = rng.choice(len(merged), size=max(1, len(merged) // 7), replace=False)
            g = np.concatenate([g, g[:3]])[::-1]
            if step == 2:
                g = np.concatenate([g, np.arange(len(merged) - 5, len(merged))])     # the tail of the last shard
            sh.remove(torch.from_numpy(g.copy()))
            drop = {merged[i] for i in g}
            for r in range(world):
                shard_pos[r] = [p for p in shard_pos[r] if p not in drop]
            for p in drop:
                del vec[p]
            alive = sorted(vec)                                # what an unsharded index given the same calls holds
            ref = np.stack([vec[p] for p in alive])
            merged = np.array([p for r in range(world) for p in shard_pos[r]], np.int64)
            ok &= sh.total == len(ref)
            sizes = [torch.zeros(1, dtype=torch.int64) for _ in range(world)]
            real_all_gather(sizes, torch.tensor([len(sh.index)]))
            ok &= [int(s) for s in sizes] == sh._sizes == [len(sp) for sp in shard_pos]
            ok &= sh.offset == sum(sh._sizes[:rank])
            q = torch.from_numpy(np.concatenate([ref[:2], rng.standard_normal((4, D)).astype(np.float32)]))
            s, i = sh.search(q, 11)
            fs, fi = flat_ref.flat_search(q.numpy(), ref, 11, "l2")
            i = i.numpy()
            expect = np.where(i >= 0, np.searchsorted(alive, merged[np.maximum(i, 0)]), -1)
            ok &= bool((expect == fi).all())                   # the merged ids name the rows the reference found
            ok &= bool((sh.to_insertion_order(i) == fi).all()) and bool(np.allclose(s.numpy(), fs, atol=1e-5))
        dist.all_gather = real_all_gather
        out[rank] = bool(ok) and not collectives           # add and remove kept offsets in step without a collective
    finally:
        dist.destroy_process_group()


def test_sharded_remove_equals_unsharded_gloo():
    world = 2
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    with mp.Manager() as m:
        out = m.dict()
        mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
        assert dict(out) == {0: True, 1: True}
