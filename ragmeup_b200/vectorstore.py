"""Vector-store drop-ins: ``Milvus`` / ``PGVector`` look-alikes over the GPU flat index
(SURVEY.md §8 rows a6-a8, a12).

Surface kept from the reference's use of langchain-milvus 0.1.3 / langchain-postgres 0.0.12:

* ``Milvus.from_documents([], embeddings, drop_old=..., connection_args={"uri": ...},
  collection_name=...)``                                   — ``server/RAGHelper.py:388-394``
* ``PGVector(embeddings=, collection_name=, connection=, use_jsonb=True)``   — ``:399-404``
* ``db.add_documents(documents, ids=ids)``                                   — ``:431``, ``:525``
* ``db.as_retriever(search_type="mmr", search_kwargs={"k": k})``             — ``:497-499``, ``:533-535``
  → retriever usable as ``retriever.invoke(q)`` and ``retriever | fn``.

Semantics kept (SURVEY Appendix A.3/A.4): Milvus-lite falls back to a FLAT index with metric L2,
returned score = squared L2 distance ascending; PGVector's default is cosine distance (1 - cos);
``search_type="mmr"`` = top-``fetch_k`` (20) by the store metric, fetch those vectors, greedy MMR
(lambda 0.5) down to k.  Result metadata carries the stored metadata plus ``pk`` (Milvus) like the
reference's stores do (``server/server.py:281-284`` reads ``source`` / ``pk``).

The corpus lives in HBM as fp32 ``[N, D]`` inside the C index; texts, ids and metadata stay on the
host.  All distance arithmetic runs in ``csrc/rmu_index.cu``.

Persistence (``vector_store_uri`` reuse, ``server/.env.template:33``, ``vector_store_initial_load``
``server/RAGHelper.py:406-434``): the reference's stores keep their rows across process restarts (a
milvus-lite file at ``connection_args["uri"]`` / a Postgres database).  Here a collection with a storage
directory appends one segment file per ``add_*`` call (vectors + ids + texts + metadata) and one per ``delete``
(the removed positions), and replays the segments in order when it is constructed again, unless ``drop_old`` is set, which deletes them.  ``Milvus``:
directory ``<uri>.b200/<collection_name>``; ``PGVector``: ``$RMU_STORE_DIR/<collection_name>`` when that
variable is set, otherwise the collection only lives in GPU memory (said once on stderr).
"""
from __future__ import annotations

import ast
import glob
import json
import os
import re
import shutil
import sys
import threading
import weakref
from typing import Any, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .documents import Document, Runnable
from .index import FlatIndex, mmr_select
from .segments import SegmentWriter, atomic_savez


_OPEN_STORES: Dict[str, "weakref.WeakSet"] = {}     # storage directory -> live stores writing segments into it


class B200Retriever(Runnable):
    """What ``VectorStore.as_retriever`` returns: ``invoke`` / ``get_relevant_documents``."""

    def __init__(self, vectorstore: "B200VectorStore", search_type: str = "similarity",
                 search_kwargs: Optional[Dict[str, Any]] = None):
        if search_type not in ("similarity", "mmr", "similarity_score_threshold"):
            raise ValueError(f"search_type of {search_type} not allowed.")
        self.vectorstore = vectorstore
        self.search_type = search_type
        self.search_kwargs = dict(search_kwargs or {})
        self.tags = [type(vectorstore).__name__]

    def _get_relevant_documents(self, query: str) -> List[Document]:
        if self.search_type == "mmr":
            return self.vectorstore.max_marginal_relevance_search(query, **self.search_kwargs)
        if self.search_type == "similarity_score_threshold":
            kw = dict(self.search_kwargs)
            thr = kw.pop("score_threshold")
            return [d for d, s in self.vectorstore.similarity_search_with_relevance_scores(query, **kw) if s >= thr]
        return self.vectorstore.similarity_search(query, **self.search_kwargs)

    def invoke(self, input: str, config: Any = None, **kwargs: Any) -> List[Document]:  # noqa: A002
        return self._get_relevant_documents(input)

    def get_relevant_documents(self, query: str, **_: Any) -> List[Document]:
        return self._get_relevant_documents(query)

    async def ainvoke(self, input: str, config: Any = None, **kwargs: Any) -> List[Document]:  # noqa: A002
        return self._get_relevant_documents(input)


class B200VectorStore:
    """Exact brute-force store on one GPU.  ``metric``: 'l2' | 'cosine' | 'ip'."""

    id_field = "pk"
    upsert_ids = False          # PGVector: adding an id that exists replaces the row; Milvus inserts a second row

    def __init__(self, embedding_function: Any, metric: str = "l2", collection_name: str = "LangChainCollection",
                 device: Optional[int] = None, storage_dir: Optional[str] = None, drop_old: bool = False):
        self.embedding_func = embedding_function
        self.metric = metric
        self.collection_name = collection_name
        self._device = device
        self.index: Optional[FlatIndex] = None
        self._pks: List[str] = []
        self._texts: List[str] = []
        self._metas: List[Dict[str, Any]] = []
        self._row_of: Dict[str, int] = {}
        self._added = 0             # rows ever inserted: default ids count them, so a deletion never makes one repeat
        self._generation = 0        # bumped by every removal: row numbers from an older generation name other documents
        self._lock = threading.RLock()
        self._storage_dir = storage_dir
        self._segments = 0
        self._segw: Optional[SegmentWriter] = None
        if storage_dir is not None:
            self._segw = SegmentWriter(self._write_segment)
            key = os.path.abspath(storage_dir)
            for other in list(_OPEN_STORES.get(key, ())):       # another store of this process may still be writing there
                other.flush()
            _OPEN_STORES.setdefault(key, weakref.WeakSet()).add(self)
            if drop_old and os.path.isdir(storage_dir):
                shutil.rmtree(storage_dir)
            self._load_segments()

    @property
    def embeddings(self) -> Any:
        """LangChain's ``VectorStore.embeddings`` (read-only there as well)."""
        return self.embedding_func

    # ------------------------------------------------------------------ construction (reference forms)
    @classmethod
    def from_documents(cls, documents: Sequence[Document], embedding: Any, **kwargs: Any) -> "B200VectorStore":
        ids = kwargs.pop("ids", None)
        store = cls(embedding, **kwargs)
        if documents:
            store.add_documents(list(documents), ids=ids)
        return store

    @classmethod
    def from_texts(cls, texts: Sequence[str], embedding: Any, metadatas: Optional[List[dict]] = None,
                   **kwargs: Any) -> "B200VectorStore":
        ids = kwargs.pop("ids", None)
        store = cls(embedding, **kwargs)
        if texts:
            store.add_texts(list(texts), metadatas=metadatas, ids=ids)
        return store

    def __len__(self) -> int:
        return len(self._pks)

    # ------------------------------------------------------------------ insert
    def _ensure_index(self, dim: int) -> FlatIndex:
        if self.index is None:
            self.index = FlatIndex(dim, self.metric, device=self._device)
        elif self.index.dim != dim:
            raise ValueError(f"embedding dimension {dim} does not match the collection ({self.index.dim})")
        return self.index

    def _insert_locked(self, vectors, texts: Sequence[str], metadatas: Sequence[dict], ids: Sequence[str]) -> None:
        """append (or, with ``upsert_ids``, replace) rows; ``self._lock`` held"""
        n = len(texts)
        index = self._ensure_index(int(vectors.shape[1]))
        new = list(range(n))
        if self.upsert_ids:
            last = {pk: j for j, pk in enumerate(ids)}                  # a batch repeating an id keeps its last row
            upd = [j for j in range(n) if ids[j] in self._row_of and last[ids[j]] == j]
            new = [j for j in range(n) if ids[j] not in self._row_of and last[ids[j]] == j]
            if upd:
                index.set_rows([self._row_of[ids[j]] for j in upd], vectors[upd])
                for j in upd:
                    r = self._row_of[ids[j]]
                    self._texts[r], self._metas[r] = texts[j], dict(metadatas[j])
        if new:
            index.add(vectors if len(new) == n else vectors[new])
            self._added += len(new)
            for j in new:
                self._row_of[ids[j]] = len(self._pks)
                self._pks.append(ids[j])
                self._texts.append(texts[j])
                self._metas.append(dict(metadatas[j]))

    def add_embeddings(self, vectors, texts: Sequence[str], metadatas: Optional[Sequence[dict]] = None,
                       ids: Optional[Sequence[str]] = None) -> List[str]:
        """Append pre-computed vectors (CUDA/CPU tensor or numpy [n, D])."""
        n = len(texts)
        if (ids is not None and len(ids) != n) or (metadatas is not None and len(metadatas) != n):
            raise ValueError("texts, metadatas and ids must have the same length")
        if n == 0:
            return []
        metas = [dict(m) for m in (metadatas or [{} for _ in range(n)])]
        texts = list(texts)
        with self._lock:                                    # default ids, rows and the host tables move together
            pks = [str(self._added + i) for i in range(n)] if ids is None else [str(i) for i in ids]
            self._insert_locked(vectors, texts, metas, pks)
            self._persist(vectors, texts, metas, pks)
        return pks

    def add_texts(self, texts: Iterable[str], metadatas: Optional[List[dict]] = None, ids: Optional[List[str]] = None,
                  batch_size: int = 1000, **_: Any) -> List[str]:
        texts = list(texts)
        out: List[str] = []
        for s in range(0, len(texts), batch_size):          # langchain-milvus inserts in chunks of 1000
            chunk = texts[s:s + batch_size]
            if hasattr(self.embedding_func, "encode_tensor"):
                vecs = self.embedding_func.encode_tensor(chunk)          # stays in HBM
            else:
                vecs = np.asarray(self.embedding_func.embed_documents(chunk), dtype=np.float32)
            out += self.add_embeddings(vecs, chunk, None if metadatas is None else metadatas[s:s + batch_size],
                                       None if ids is None else ids[s:s + batch_size])
        return out

    def add_documents(self, documents: List[Document], ids: Optional[List[str]] = None, **kwargs: Any) -> List[str]:
        texts = [d.page_content for d in documents]
        metas = [d.metadata for d in documents]
        return self.add_texts(texts, metas, ids=ids, **kwargs)

    # ------------------------------------------------------------------ delete
    def _remove_locked(self, rows: Sequence[int]) -> int:
        """remove rows (positions, any order) from the index and the host tables in one pass; ``self._lock`` held"""
        drop = set(int(r) for r in rows)
        if not drop:
            return 0
        self.index.remove(sorted(drop))
        keep = [r for r in range(len(self._pks)) if r not in drop]
        self._pks = [self._pks[r] for r in keep]
        self._texts = [self._texts[r] for r in keep]
        self._metas = [self._metas[r] for r in keep]
        self._row_of = {pk: r for r, pk in enumerate(self._pks)}    # a repeated pk maps to its last row, as after adds
        self._generation += 1
        return len(drop)

    def _delete_rows(self, match) -> int:
        """remove every row r with ``match(r)``; persisted as the removed positions, through the segment writer"""
        with self._lock:
            rows = [r for r in range(len(self._pks)) if match(r)]
            if not rows:
                return 0
            self._remove_locked(rows)
            self._persist(None, [], [], [], deleted=rows)
        return len(rows)

    def _delete_by_ids(self, ids: Iterable[Any]) -> int:
        want = set(str(i) for i in ids)
        return self._delete_rows(lambda r: self._pks[r] in want)

    def delete(self, ids: Optional[Sequence[Any]] = None, expr: Optional[str] = None, **_: Any) -> "DeleteResult":
        """``langchain_milvus.Milvus.delete`` (``PGVector`` narrows it to ids): every row whose pk is in ``ids`` (then
        ``expr`` is ignored, as langchain-milvus does), or every row ``expr`` matches.  ``expr`` takes the forms the reference writes,
        ``<field> == "<string>"`` and ``<field> in ["a", ...]``, where the field is ``pk`` or a metadata key
        (``db.delete(expr='source == "<path>"')`` removes a file's chunks).  Any other expression raises ``ValueError``
        and deletes nothing.  The result's ``delete_count`` is the number of rows removed."""
        if ids is not None and len(ids) > 0:
            return DeleteResult(self._delete_by_ids(ids))
        if not isinstance(expr, str):
            raise ValueError("Either ids list or expr string must be provided.")
        field, values = parse_delete_expr(expr)
        if field == self.id_field:
            return DeleteResult(self._delete_by_ids(values))
        return DeleteResult(self._delete_rows(lambda r: self._metas[r].get(field, _NO_VALUE) in values))

    # ------------------------------------------------------------------ persistence: one segment per add call
    # written in order by the store's SegmentWriter (segments.py); ``flush()`` runs in ``save`` and before segments are
    # re-read
    @property
    def _writer(self):
        """the background writer thread, None until the first asynchronous segment"""
        return self._segw.thread if self._segw is not None else None

    def _persist(self, vectors, texts, metas, pks, deleted: Optional[List[int]] = None,
                 added: Optional[int] = None) -> None:
        """queue the next segment; ``self._lock`` held"""
        if self._storage_dir is None:
            return
        seg = self._segments
        self._segments += 1
        self._segw.submit(seg, vectors, list(texts), [dict(m) for m in metas], list(pks), deleted, added)

    def flush(self) -> None:
        """Wait until every segment queued so far is on disk."""
        if self._segw is not None:
            self._segw.flush()

    def _write_segment(self, seg: int, vectors, texts, metas, pks, deleted: Optional[List[int]] = None,
                       added: Optional[int] = None) -> None:
        """an add segment; with ``deleted`` a deletion record: the positions removed, as they were at that moment (pks
        would not do: Milvus keeps repeated pks, and an expression may match only some of those rows); with ``added``
        the default-id counter carried over from an export"""
        os.makedirs(self._storage_dir, exist_ok=True)
        if added is not None:
            vec = np.zeros((0, 0), np.float32)
            table = np.frombuffer(json.dumps({"added": int(added)}).encode(), dtype=np.uint8)
        elif deleted is not None:
            vec = np.zeros((0, 0), np.float32)
            table = np.frombuffer(json.dumps({"deleted": [int(r) for r in deleted]}).encode(), dtype=np.uint8)
        else:
            vec = vectors if isinstance(vectors, np.ndarray) else vectors.detach().float().cpu().numpy()
            table = np.frombuffer(json.dumps({"pks": pks, "texts": texts, "metas": metas}).encode(), dtype=np.uint8)
        atomic_savez(os.path.join(self._storage_dir, f"seg_{seg:08d}.npz"),
                     vectors=np.ascontiguousarray(vec, dtype=np.float32), metric=self.metric, table=table)

    def _load_segments(self) -> None:
        files = sorted(glob.glob(os.path.join(self._storage_dir, "seg_*.npz")))
        files = [f for f in files if not f.endswith(".tmp.npz")]
        for f in files:
            z = np.load(f, allow_pickle=False)
            if str(z["metric"]) != self.metric:
                raise ValueError(f"{f} was written by a {z['metric']} collection, this store is {self.metric}")
            table = json.loads(bytes(z["table"]).decode())
            if "deleted" in table:                          # replayed in order: positions refer to the rows at that point
                with self._lock:
                    self._remove_locked(table["deleted"])
            elif "added" in table:
                with self._lock:
                    self._added = max(self._added, int(table["added"]))
            elif z["vectors"].size:
                with self._lock:
                    self._insert_locked(np.ascontiguousarray(z["vectors"]), table["texts"], table["metas"], table["pks"])
        self._segments = len(files)

    # ------------------------------------------------------------------ search (tensor level)
    def _score_out(self, scores):
        """index metric value -> the score the reference's store reports"""
        return (1.0 - scores) if self.metric == "cosine" else scores

    def search_tensor(self, queries, k: int):
        """CUDA fp32 [Q, D] -> (scores [Q,k], rows int64 [Q,k]) on the device; rows index insertion order.  A delete
        renumbers the rows above the first one it removes: a caller that may race with one holds ``self._lock``."""
        if self.index is None:
            raise _lib.RmuError("the collection is empty")
        s, i = self.index.search(queries, k)
        return self._score_out(s), i

    def mmr_tensor(self, queries, k: int = 4, fetch_k: int = 20, lambda_mult: float = 0.5):
        """CUDA fp32 [Q, D] -> rows int64 [Q, k] in MMR order (-1 padded), all on the device (rows as in
        :meth:`search_tensor`)."""
        if self.index is None:
            raise _lib.RmuError("the collection is empty")
        torch = self.index.torch
        q = queries.to(device=self.index.device, dtype=torch.float32).contiguous()
        _, rows = self.index.search(q, fetch_k)
        n_cand = (rows >= 0).sum(1).to(torch.int32)
        cand = self.index.gather(rows.clamp_min(0).view(-1)).view(q.shape[0], fetch_k, self.index.dim)
        sel = mmr_select(q, cand, n_cand, k, lambda_mult).to(torch.int64)
        picked = torch.gather(rows, 1, sel.clamp_min(0))
        return torch.where(sel >= 0, picked, torch.full_like(picked, -1))

    # ------------------------------------------------------------------ search (reference surface)
    def _doc(self, row: int) -> Document:
        meta = dict(self._metas[row])
        meta[self.id_field] = self._pks[row]
        return Document(page_content=self._texts[row], metadata=meta)

    def _docs(self, rows: Sequence[int], scores: Optional[Sequence[float]] = None):
        """rows -> documents; an insert may be between index.add and the host tables, so wait for it"""
        with self._lock:
            if scores is None:
                return [self._doc(r) for r in rows if r >= 0]
            return [(self._doc(r), float(sc)) for sc, r in zip(scores, rows) if r >= 0]

    def _search_docs(self, run, with_scores: bool):
        """``run()`` searches the device -> (rows, scores) of query 0 as lists -> documents.  The search runs outside the
        lock, so that searches do not wait for each other's host work.  A delete that lands between the search and the
        mapping renumbers the rows, so then the search runs again under the lock, where no delete can interleave."""
        gen = self._generation
        rows, scores = run()
        with self._lock:
            if gen != self._generation:
                rows, scores = run()
            return self._docs(rows, scores if with_scores else None)

    def _embed_query_tensor(self, query: str):
        torch = _lib.require_cuda()
        if hasattr(self.embedding_func, "encode_tensor"):
            return self.embedding_func.encode_tensor([query])
        return torch.tensor([self.embedding_func.embed_query(query)], dtype=torch.float32, device="cuda")

    def _top_rows(self, q, k: int):
        s, i = self.search_tensor(q, k)
        return i[0].tolist(), s[0].tolist()

    def similarity_search_with_score_by_vector(self, embedding: List[float], k: int = 4, **_: Any) -> List[Tuple[Document, float]]:
        if self.index is None or len(self) == 0:
            return []
        torch = self.index.torch
        q = torch.as_tensor(np.asarray(embedding, dtype=np.float32)[None], device=self.index.device)
        return self._search_docs(lambda: self._top_rows(q, k), True)

    def similarity_search_with_score(self, query: str, k: int = 4, **kw: Any) -> List[Tuple[Document, float]]:
        if self.index is None or len(self) == 0:
            return []
        q = self._embed_query_tensor(query)
        return self._search_docs(lambda: self._top_rows(q, k), True)

    def similarity_search(self, query: str, k: int = 4, **kw: Any) -> List[Document]:
        return [d for d, _ in self.similarity_search_with_score(query, k, **kw)]

    def similarity_search_by_vector(self, embedding: List[float], k: int = 4, **kw: Any) -> List[Document]:
        return [d for d, _ in self.similarity_search_with_score_by_vector(embedding, k, **kw)]

    def similarity_search_with_relevance_scores(self, query: str, k: int = 4, **kw: Any) -> List[Tuple[Document, float]]:
        out = []
        for d, s in self.similarity_search_with_score(query, k, **kw):
            if self.metric == "l2":
                rel = 1.0 - s / 2.0 ** 0.5          # LangChain's euclidean relevance for unit vectors
            elif self.metric == "cosine":
                rel = 1.0 - s
            else:
                rel = s
            out.append((d, rel))
        return out

    def max_marginal_relevance_search_by_vector(self, embedding: List[float], k: int = 4, fetch_k: int = 20,
                                                lambda_mult: float = 0.5, **_: Any) -> List[Document]:
        if self.index is None or len(self) == 0:
            return []
        torch = self.index.torch
        q = torch.as_tensor(np.asarray(embedding, dtype=np.float32)[None], device=self.index.device)
        return self._search_docs(lambda: (self.mmr_tensor(q, k, fetch_k, lambda_mult)[0].tolist(), None), False)

    def max_marginal_relevance_search(self, query: str, k: int = 4, fetch_k: int = 20, lambda_mult: float = 0.5,
                                      **_: Any) -> List[Document]:
        if self.index is None or len(self) == 0:
            return []
        q = self._embed_query_tensor(query)
        return self._search_docs(lambda: (self.mmr_tensor(q, k, fetch_k, lambda_mult)[0].tolist(), None), False)

    def as_retriever(self, **kwargs: Any) -> B200Retriever:
        return B200Retriever(self, kwargs.get("search_type", "similarity"), kwargs.get("search_kwargs"))

    # ------------------------------------------------------------------ one-file export / import
    def save(self, path: str) -> None:
        """the whole collection as one ``.npz`` (an export; the segment directory is the live persistence)"""
        self.flush()
        with self._lock:
            vec = self.index.data().cpu().numpy() if self.index is not None else np.zeros((0, 0), np.float32)
            table = json.dumps({"pks": self._pks, "texts": self._texts, "metas": self._metas, "added": self._added}).encode()
        np.savez(path, vectors=vec, metric=self.metric, table=np.frombuffer(table, dtype=np.uint8))

    @classmethod
    def load(cls, path: str, embedding: Any, **kwargs: Any) -> "B200VectorStore":
        z = np.load(path if path.endswith(".npz") else path + ".npz", allow_pickle=False)
        store = cls(embedding, **kwargs)
        if str(z["metric"]) != store.metric:
            raise ValueError(f"{path} holds a {z['metric']} collection, {cls.__name__} searches with {store.metric}")
        table = json.loads(bytes(z["table"]).decode())
        if z["vectors"].size:
            store.add_embeddings(np.ascontiguousarray(z["vectors"]), table["texts"], table["metas"], table["pks"])
        store._restore_added(int(table.get("added", 0)))
        return store

    def _restore_added(self, added: int) -> None:
        """default ids keep counting past rows deleted before an export; a storage directory records the counter too"""
        with self._lock:
            if added <= self._added:
                return
            self._added = added
            self._persist(None, [], [], [], added=added)


class Milvus(B200VectorStore):
    """Answers to ``langchain_milvus.vectorstores.Milvus`` as constructed at
    ``server/RAGHelper.py:388-394`` (FLAT / L2).  ``connection_args["uri"]`` (the milvus-lite file of the
    reference, ``vector_store_uri``) names where the collection persists: ``<uri>.b200/<collection_name>``;
    ``drop_old=True`` deletes what is stored there, otherwise it is loaded."""

    def __init__(self, embedding_function: Any, collection_name: str = "LangChainCollection",
                 connection_args: Optional[Dict[str, Any]] = None, drop_old: bool = False, auto_id: bool = False,
                 device: Optional[int] = None, **_: Any):
        self.connection_args = dict(connection_args or {})
        self.drop_old = drop_old
        self.auto_id = auto_id
        uri = self.connection_args.get("uri")
        storage = None
        if uri and "://" not in str(uri):                   # a local path, as the reference configures milvus-lite
            storage = os.path.join(str(uri) + ".b200", collection_name)
        super().__init__(embedding_function, metric="l2", collection_name=collection_name, device=device,
                         storage_dir=storage, drop_old=drop_old)


class DeleteResult:
    """what ``pymilvus`` ``Collection.delete`` returns, as far as the reference reads it (``delete_count``)"""

    def __init__(self, delete_count: int):
        self.delete_count = int(delete_count)

    def __repr__(self) -> str:
        return f"(delete count: {self.delete_count})"


_NO_VALUE = object()
_EXPR = re.compile(r"^\s*([A-Za-z_][A-Za-z0-9_]*)\s*(==|\bin\b)\s*(.+?)\s*$", re.S)


def parse_delete_expr(expr: str) -> Tuple[str, List[str]]:
    """``<field> == "<string>"`` / ``<field> in ["a", ...]`` (quoted strings, single or double quotes) ->
    (field, [values]); anything else raises ``ValueError``."""
    m = _EXPR.match(expr)
    if m is None:
        raise ValueError(f"unsupported delete expression {expr!r}: use <field> == \"<string>\" or <field> in [\"a\", ...]")
    field, op, rhs = m.groups()
    try:
        value = ast.literal_eval(rhs)
    except (ValueError, SyntaxError):
        value = None
    if op == "==" and isinstance(value, str) and rhs[0] in "'\"":
        return field, [value]
    if op == "in" and isinstance(value, list) and rhs[0] == "[" and all(isinstance(v, str) for v in value):
        return field, list(value)
    raise ValueError(f"unsupported delete expression {expr!r}: use <field> == \"<string>\" or <field> in [\"a\", ...]")


_warned_memory_only = False


class PGVector(B200VectorStore):
    """Answers to ``langchain_postgres.vectorstores.PGVector`` as constructed at
    ``server/RAGHelper.py:399-404`` (default distance strategy COSINE, score = 1 - cos; adding an id that
    exists replaces the row).  There is no Postgres behind it: rows persist under ``$RMU_STORE_DIR`` when set."""

    id_field = "id"
    upsert_ids = True

    def __init__(self, embeddings: Any = None, collection_name: str = "langchain", connection: Any = None,
                 use_jsonb: bool = True, pre_delete_collection: bool = False, device: Optional[int] = None, **_: Any):
        global _warned_memory_only
        self.connection = connection
        self.use_jsonb = use_jsonb
        root = os.environ.get("RMU_STORE_DIR")
        if not root and not _warned_memory_only:
            print("ragmeup_b200.PGVector: RMU_STORE_DIR is not set, the collection lives in GPU memory only "
                  "(rows are not kept across restarts)", file=sys.stderr)
            _warned_memory_only = True
        super().__init__(embeddings, metric="cosine", collection_name=collection_name, device=device,
                         storage_dir=os.path.join(root, collection_name) if root else None, drop_old=pre_delete_collection)

    def delete(self, ids: Optional[Sequence[Any]] = None, collection_only: bool = False, **_: Any) -> None:
        """``langchain_postgres.PGVector.delete``: removes the row of each id; unknown ids are ignored."""
        if ids:
            self._delete_by_ids(ids)
