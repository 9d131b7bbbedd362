"""CPU: deleting documents from the vector-store drop-ins (``Milvus.delete`` by ids and by the expressions the
reference writes, ``PGVector.delete``), default ids after a deletion, and deletions surviving a reload, with the CUDA
index replaced by a numpy stand-in that has ``remove``."""
import threading

import numpy as np
import pytest

from oracle import flat_ref
from ragmeup_b200 import vectorstore as vs
from ragmeup_b200.documents import Document


class RemovableIndex:
    """FlatIndex look-alike with ``remove`` (the product index needs a GPU; only the host logic is under test)."""

    def __init__(self, dim, metric, device=None):
        import torch
        self.dim, self.metric, self.device, self.torch = dim, metric, "cpu", torch
        self.x = np.zeros((0, dim), np.float32)

    def __len__(self):
        return len(self.x)

    def add(self, v):
        self.x = np.concatenate([self.x, np.asarray(v, np.float32)])

    def set_rows(self, rows, v):
        self.x[np.asarray(rows)] = np.asarray(v, np.float32)

    def remove(self, rows):
        rows = np.asarray(rows, np.int64)
        assert rows.size == 0 or (rows.min() >= 0 and rows.max() < len(self.x))
        self.x = np.delete(self.x, rows, axis=0)

    def gather(self, rows):
        r = np.asarray(rows.cpu() if hasattr(rows, "cpu") else rows, np.int64)
        ok = (r >= 0) & (r < len(self.x))
        out = np.zeros((len(r), self.dim), np.float32)
        out[ok] = self.x[r[ok]]
        return self.torch.from_numpy(out)

    def search(self, q, k, **_):
        import torch
        s, i = flat_ref.flat_search(np.asarray(q.cpu() if hasattr(q, "cpu") else q, np.float32), self.x, k, self.metric)
        return torch.from_numpy(s), torch.from_numpy(i)


class Emb:
    def embed_documents(self, texts):
        return [[float(len(t)), float(sum(map(ord, t)) % 7), 1.0] for t in texts]

    def embed_query(self, t):
        return self.embed_documents([t])[0]


@pytest.fixture()
def numpy_index(monkeypatch):
    monkeypatch.setattr(vs, "FlatIndex", RemovableIndex)


def _docs(n, off=0, source=None):
    return [Document(f"text {i + off}" * (1 + i % 3), {"source": source or f"s{i + off}"}) for i in range(n)]


def _state(st):
    return list(st._pks), list(st._texts), [dict(m) for m in st._metas], st.index.x.copy()


def _consistent(st):
    assert len(st.index) == len(st._pks) == len(st._texts) == len(st._metas)
    assert st._row_of == {pk: r for r, pk in enumerate(st._pks)}


def test_milvus_delete_by_ids_takes_every_row_of_a_pk(numpy_index):
    m = vs.Milvus(Emb())
    m.add_documents(_docs(4), ids=["a", "b", "c", "d"])
    m.add_documents(_docs(2, 10), ids=["b", "e"])                # Milvus keeps a second row with pk b
    x = m.index.x.copy()
    res = m.delete(ids=["b", "zz"])
    assert res.delete_count == 2
    assert m._pks == ["a", "c", "d", "e"] and m._texts == [d.page_content for d in (_docs(4)[0], *_docs(4)[2:], _docs(2, 10)[1])]
    assert np.array_equal(m.index.x, x[[0, 2, 3, 5]])
    _consistent(m)
    assert m.delete(ids=["nope"]).delete_count == 0              # unknown ids delete nothing
    assert len(m) == 4


def test_milvus_delete_by_expression(numpy_index):
    m = vs.Milvus(Emb())
    m.add_documents(_docs(3, source="a.pdf") + _docs(2, 3) + _docs(2, 5, source="b.pdf"), ids=list("pqrstuv"))
    assert m.delete(expr='source == "a.pdf"').delete_count == 3
    assert m._pks == list("stuv")
    assert m.delete(expr="source in ['b.pdf', 's3']").delete_count == 3
    assert m._pks == ["t"]
    m.add_documents(_docs(3), ids=["x", "y", "t"])
    assert m.delete(expr='pk == "t"').delete_count == 2
    assert m.delete(expr='pk in ["x", "nope"]').delete_count == 1
    assert m._pks == ["y"]
    _consistent(m)
    assert m.delete(ids=["y"], expr='pk == "nope"').delete_count == 1      # ids win over expr


@pytest.mark.parametrize("expr", ['source != "a.pdf"', "source == 3", 'source == "a.pdf" or pk == "p"', "pk in [1, 2]",
                                  'source like "a%"', "", 'source in "a.pdf"'])
def test_refused_expressions_delete_nothing(numpy_index, expr):
    m = vs.Milvus(Emb())
    m.add_documents(_docs(3, source="a.pdf"), ids=["p", "q", "r"])
    with pytest.raises(ValueError):
        m.delete(expr=expr)
    assert m._pks == ["p", "q", "r"] and len(m.index) == 3
    with pytest.raises(ValueError):
        m.delete()


def test_pgvector_delete(numpy_index, tmp_path, monkeypatch):
    monkeypatch.setenv("RMU_STORE_DIR", str(tmp_path / "pg"))
    pg = vs.PGVector(embeddings=Emb(), collection_name="c", connection="postgresql://x")
    pg.add_documents(_docs(4), ids=["a", "b", "c", "d"])
    assert pg.delete(["b", "d", "zz"]) is None
    assert pg._pks == ["a", "c"] and pg._row_of == {"a": 0, "c": 1}
    pg.add_documents([Document("new c", {})], ids=["c"])          # the upsert still finds the moved row
    assert pg._texts == [_docs(4)[0].page_content, "new c"] and len(pg.index) == 2
    again = vs.PGVector(embeddings=Emb(), collection_name="c", connection="postgresql://x")
    assert again._pks == ["a", "c"] and again._texts == pg._texts and np.array_equal(again.index.x, pg.index.x)


def test_default_ids_stay_unique_after_a_delete(numpy_index):
    m = vs.Milvus(Emb())
    first = m.add_texts(["a", "bb", "ccc"])
    assert first == ["0", "1", "2"]                              # unchanged while nothing was deleted
    m.delete(ids=["0"])
    more = m.add_texts(["dddd"])
    assert more == ["3"] and len(set(m._pks)) == len(m._pks)


@pytest.mark.parametrize("sync", ["0", "1"])
def test_live_state_equals_reloaded_state(numpy_index, tmp_path, monkeypatch, sync):
    monkeypatch.setenv("RMU_STORE_SYNC", sync)
    uri = str(tmp_path / "data.db")
    m = vs.Milvus(Emb(), connection_args={"uri": uri}, drop_old=True)
    m.add_documents(_docs(6, source="f1") + _docs(4, 6), ids=[f"id{i % 7}" for i in range(10)])
    m.delete(expr='source == "f1"')
    m.add_documents(_docs(5, 20, source="f2"), ids=["id1", "n1", "n2", "n3", "n4"])   # id1 repeats a pk kept from before
    m.delete(expr='source in ["f2", "s7"]')        # only some of the rows with pk id1: replay must use positions
    m.add_texts(["tail"])
    m.flush()
    live = _state(m)
    back = vs.Milvus(Emb(), connection_args={"uri": uri})
    got = _state(back)
    assert got[:3] == live[:3] and np.array_equal(got[3], live[3])
    _consistent(back)
    assert back._added == m._added                               # the default-id counter survives the reload too
    dropped = vs.Milvus(Emb(), connection_args={"uri": uri}, drop_old=True)
    assert len(dropped) == 0


def test_search_after_delete_maps_to_the_right_texts(numpy_index):
    m = vs.Milvus(Emb())
    docs = _docs(8)
    m.add_documents(docs, ids=[f"k{i}" for i in range(8)])
    m.delete(ids=["k0", "k3", "k4"])
    kept = [docs[i] for i in (1, 2, 5, 6, 7)]
    for d in kept:
        got = m.similarity_search_by_vector(Emb().embed_query(d.page_content), k=1)
        assert got[0].page_content == d.page_content and got[0].metadata["source"] == d.metadata["source"]
    res = m.similarity_search_with_score_by_vector(Emb().embed_query(docs[3].page_content), k=5)
    assert len(res) == 5 and all(d.metadata["pk"] in {"k1", "k2", "k5", "k6", "k7"} for d, _ in res)
    for d, _ in res:
        r = m._row_of[d.metadata["pk"]]
        assert m._texts[r] == d.page_content


def test_save_and_load_after_delete(numpy_index, tmp_path, monkeypatch):
    m = vs.Milvus(Emb())
    m.add_documents(_docs(5), ids=list("abcde"))
    m.delete(ids=["b"])
    assert m.add_texts(["x", "y"]) == ["5", "6"]
    m.delete(ids=["a", "6"])
    m.index.data = lambda: type("T", (), {"cpu": lambda self: type("N", (), {"numpy": lambda s: m.index.x})()})()
    m.save(str(tmp_path / "one.npz"))
    back = vs.Milvus.load(str(tmp_path / "one.npz"), Emb())
    assert back._pks == list("cde") + ["5"] and np.array_equal(back.index.x, m.index.x)
    assert back.add_texts(["z"]) == ["7"]                        # the default-id counter travels with the export
    # loaded into a collection with a storage directory, the counter also survives the next restart
    monkeypatch.setenv("RMU_STORE_SYNC", "1")
    uri = str(tmp_path / "data.db")
    kept = vs.Milvus.load(str(tmp_path / "one.npz"), Emb(), connection_args={"uri": uri}, drop_old=True)
    assert kept._added == 7
    again = vs.Milvus(Emb(), connection_args={"uri": uri})
    assert again._pks == kept._pks and again.add_texts(["w"]) == ["7"]


@pytest.mark.parametrize("kind", ["similarity", "mmr"])
def test_delete_between_search_and_mapping(numpy_index, monkeypatch, kind):
    """A delete from another thread (the /delete endpoint while a /chat request is in flight) that lands after the
    device search and before its rows are mapped to documents renumbers the rows: the search still returns the
    document it scored."""
    import torch
    monkeypatch.setattr(vs, "mmr_select", lambda q, cand, n_cand, k, lam=0.5:
                        torch.arange(k, dtype=torch.int32).expand(q.shape[0], k).clone())   # MMR order = score order
    m = vs.Milvus(Emb())
    docs = _docs(8)
    m.add_documents(docs, ids=[f"k{i}" for i in range(8)])
    real_search = m.index.search
    deleted = []

    def search_then_delete(q, k, **kw):
        out = real_search(q, k, **kw)
        if not deleted:                                  # once: the delete runs to completion between search and mapping
            t = threading.Thread(target=lambda: deleted.append(m.delete(ids=["k0", "k2"]).delete_count))
            t.start()
            t.join(5)
            assert deleted == [2]                        # the delete did not wait for the search
        return out
    m.index.search = search_then_delete
    target = docs[5]
    emb = Emb().embed_query(target.page_content)
    if kind == "mmr":
        got = m.max_marginal_relevance_search_by_vector(emb, k=1, fetch_k=3)
    else:
        got = [d for d, _ in m.similarity_search_with_score_by_vector(emb, k=1)]
    assert len(got) == 1 and got[0].page_content == target.page_content and got[0].metadata["pk"] == "k5"
