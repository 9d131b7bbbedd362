"""PostgresBM25Retriever: the reference's pg_search sparse leg, scored on the GPU.

Stands where ``server/PostgresBM25Retriever.py`` stands for ``vector_store=postgres`` (``server/RAGHelper.py:32``,
built at ``:445-462``, fed at ``:468-469`` and ``:527-528``, fused at ``:501-503``), without a Postgres server:
``connection_uri`` is ignored and psycopg2 is never imported.

* ``PgTable`` is the reference's table ``id SERIAL PRIMARY KEY, hash char(32) UNIQUE, content TEXT, metadata TEXT``
  on the host: ``INSERT ... ON CONFLICT (hash) DO NOTHING`` row by row (a skipped row still uses up a SERIAL id), ids
  longer than 32 characters refused, metadata as ``json.dumps`` text, deletes by SERIAL id.  Rows persist under
  ``$RMU_STORE_DIR/<table_name>/`` when that variable is set (one segment per change, through the vector store's
  ``SegmentWriter``), otherwise in memory only.
* ``PgBM25Index`` is the BM25 index over ``content`` on the device: rows are tokenized on add and collect on the host;
  at the next search they become an immutable device segment, and trailing segments merge geometrically (a segment
  is at least twice the size of the next), so a corpus holds O(log N) segments.  Deletes clear bits of an alive
  bitmap; the statistics (N, average length, document frequencies) are always those of the live rows, as after the
  reference's ``VACUUM``.  Scoring and top-k run in ``csrc/rmu_pgbm25.cu``; the rules are in ``pg_search.py``.
"""
from __future__ import annotations

import ctypes as C
import glob
import json
import os
import sys
import threading
import uuid
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib, pg_search
from .documents import Document
from .retrievers import _Retriever
from .segments import SegmentWriter, atomic_savez

MAX_K = 256
HASH_CHARS = 32                 # hash char(32)


def _ptr(a: np.ndarray) -> int:
    return a.ctypes.data


class PgBM25Index:
    """Appendable inverted index with positions over rows 0, 1, ... (insertion order), searched on the device."""

    def __init__(self, device: Optional[int] = None):
        torch = _lib.require_cuda()
        self.torch = torch
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_pgbm25_create(C.byref(self._h)), "rmu_pgbm25_create")
        self.vocab: Dict[str, int] = {}
        self._df = np.zeros(1024, dtype=np.int64)         # live document frequency per term id
        self._lens: List[int] = []                        # tokens per row
        self._alive = np.zeros(0, dtype=bool)
        self.n_live = 0
        self.total_live = 0                               # tokens over the live rows
        self._pending: List[Tuple[np.ndarray, np.ndarray]] = []    # (term ids, positions) of rows not yet on the device
        self._segs: List[Dict[str, Any]] = []             # host copies of the device segments, in row order
        self._alive_dirty = True

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                _lib.lib().rmu_pgbm25_destroy(h)
            except Exception:
                pass
            self._h = C.c_void_p()

    def __len__(self) -> int:
        return len(self._lens)

    def segments(self) -> int:
        return int(_lib.lib().rmu_pgbm25_segments(self._h))

    # ---------------------------------------------------------------------------------------------- rows
    def _terms(self, text: str) -> Tuple[List[int], List[int]]:
        toks, pos = pg_search.tokenize(text)
        vocab = self.vocab
        ids = []
        for t in toks:
            i = vocab.get(t)
            if i is None:
                i = vocab[t] = len(vocab)
            ids.append(i)
        return ids, pos

    def add(self, text: str) -> int:
        """append one row; returns its row number"""
        ids, pos = self._terms(text)
        if len(self.vocab) > len(self._df):
            self._df = np.concatenate([self._df, np.zeros(max(len(self.vocab), 2 * len(self._df)) - len(self._df), np.int64)])
        uniq = np.unique(np.asarray(ids, dtype=np.int64))
        self._df[uniq] += 1
        row = len(self._lens)
        self._lens.append(len(ids))
        self.n_live += 1
        self.total_live += len(ids)
        self._pending.append((np.asarray(ids, dtype=np.int32), np.asarray(pos, dtype=np.int32)))
        self._alive_dirty = True
        return row

    def delete(self, row: int, text: str) -> None:
        """mark a live row dead; ``text`` is its content (its terms leave the document frequencies)"""
        if row >= len(self._alive):
            self._grow_alive()
        if not self._alive[row]:
            return
        self._alive[row] = False
        ids = np.unique(np.asarray([self.vocab[t] for t in pg_search.tokenize(text)[0]], dtype=np.int64))
        self._df[ids] -= 1
        self.n_live -= 1
        self.total_live -= self._lens[row]
        self._alive_dirty = True

    def _grow_alive(self) -> None:
        n = len(self._lens)
        if n > len(self._alive):
            self._alive = np.concatenate([self._alive, np.ones(n - len(self._alive), dtype=bool)])

    # ---------------------------------------------------------------------------------------------- device segments
    @staticmethod
    def _segment(row0: int, n_rows: int, n_terms: int, tok_term, tok_row, tok_pos, fnorm) -> Dict[str, Any]:
        """CSR by term from token triples in row order (positions ascending inside a row)"""
        order = np.argsort(tok_term, kind="stable")       # rows, then positions, stay ascending inside a term
        t, r, p = tok_term[order], tok_row[order], tok_pos[order]
        new = np.ones(len(t), dtype=bool)
        new[1:] = (t[1:] != t[:-1]) | (r[1:] != r[:-1])
        starts = np.flatnonzero(new)
        post_tf = np.diff(np.append(starts, len(t))).astype(np.int32)
        post_ptr = np.zeros(n_terms + 1, dtype=np.int64)
        np.cumsum(np.bincount(t[starts], minlength=n_terms), out=post_ptr[1:])
        return dict(row0=row0, n_rows=n_rows, n_terms=n_terms, post_ptr=post_ptr,
                    post_row=np.ascontiguousarray(r[starts], dtype=np.int32), post_tf=post_tf,
                    pos_start=starts.astype(np.int64), pos=np.ascontiguousarray(p, dtype=np.int32),
                    fnorm=np.ascontiguousarray(fnorm, dtype=np.uint8))

    @staticmethod
    def _tokens(seg: Dict[str, Any], row0: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        terms = np.repeat(np.arange(seg["n_terms"], dtype=np.int64), np.diff(seg["post_ptr"]))
        return (np.repeat(terms, seg["post_tf"]), np.repeat(seg["post_row"].astype(np.int64) + seg["row0"] - row0,
                                                            seg["post_tf"]), seg["pos"])

    def _push(self, seg: Dict[str, Any]) -> None:
        _lib.check(_lib.lib().rmu_pgbm25_push_segment(
            self._h, seg["row0"], seg["n_rows"], seg["n_terms"], _ptr(seg["post_ptr"]), _ptr(seg["post_row"]),
            _ptr(seg["post_tf"]), _ptr(seg["pos_start"]), _ptr(seg["pos"]), _ptr(seg["fnorm"])), "rmu_pgbm25_push_segment")
        self._segs.append(seg)

    def flush(self) -> None:
        """pending rows -> one device segment, merged with the trailing segments it is not half the size of; then the
        alive bitmap"""
        with self.torch.cuda.device(self.device):
            if self._pending:
                row0 = len(self._lens) - len(self._pending)
                ids = [a for a, _ in self._pending]
                counts = np.asarray([len(a) for a in ids], dtype=np.int64)
                tok_term = np.concatenate(ids).astype(np.int64) if ids else np.zeros(0, np.int64)
                tok_pos = np.concatenate([p for _, p in self._pending])
                tok_row = np.repeat(np.arange(len(ids), dtype=np.int64), counts)
                fnorm = pg_search.fieldnorm_id(self._lens[row0:])
                seg = self._segment(row0, len(ids), len(self.vocab), tok_term, tok_row, tok_pos, fnorm)
                self._pending = []
                merge = [seg]
                while self._segs and self._segs[-1]["n_rows"] < 2 * sum(s["n_rows"] for s in merge):
                    merge.insert(0, self._segs.pop())
                if len(merge) > 1:
                    _lib.check(_lib.lib().rmu_pgbm25_pop_segments(self._h, len(merge) - 1), "rmu_pgbm25_pop_segments")
                    r0 = merge[0]["row0"]
                    parts = [self._tokens(s, r0) for s in merge]
                    seg = self._segment(r0, sum(s["n_rows"] for s in merge), len(self.vocab),
                                        np.concatenate([a for a, _, _ in parts]), np.concatenate([b for _, b, _ in parts]),
                                        np.concatenate([c for _, _, c in parts]), np.concatenate([s["fnorm"] for s in merge]))
                self._push(seg)
            if self._alive_dirty:
                self._grow_alive()
                words = np.packbits(self._alive, bitorder="little")
                words = np.concatenate([words, np.zeros((-len(words)) % 4, np.uint8)]).view(np.uint32)
                _lib.check(_lib.lib().rmu_pgbm25_set_alive(self._h, _ptr(words), len(words)), "rmu_pgbm25_set_alive")
                self._alive_dirty = False

    # ---------------------------------------------------------------------------------------------- search
    def search(self, queries: Sequence[List[pg_search.Clause]], k: int) -> Tuple[np.ndarray, np.ndarray]:
        """parsed queries -> (float32 scores [Q, k], int64 rows [Q, k]), score descending, ties by lower row, -1 past the
        matches"""
        if k < 1:
            raise ValueError("k must be >= 1")
        if k > MAX_K:
            raise _lib.RmuError(f"PgBM25Index.search: k={k} exceeds {MAX_K}")
        nq = len(queries)
        scores = np.zeros((nq, k), dtype=np.float32)
        rows = np.full((nq, k), -1, dtype=np.int64)
        if nq == 0:
            return scores, rows
        self.flush()
        n = self.n_live
        q_ptr, occ, wts, tptr, terms, offs = [0], [], [], [0], [], []
        for clauses in queries:
            enc = []
            for c in clauses:
                if len(c.tokens) > 128:
                    raise ValueError("pg_search query: a phrase of more than 128 tokens is not supported")
                ids = [self.vocab.get(t) for t in c.tokens]
                df = [int(self._df[i]) if i is not None else 0 for i in ids]
                if min(df) == 0:                          # matches no live row
                    if c.occur == pg_search.MUST:
                        enc = []                          # the whole query matches nothing
                        break
                    continue
                w = pg_search.clause_weight(pg_search.idf(df, n)) if c.occur != pg_search.MUST_NOT else np.float32(0)
                order = sorted(range(len(ids)), key=lambda j: df[j])      # the rarest term drives a phrase
                enc.append((c.occur, w, [ids[j] for j in order], [c.offsets[j] for j in order]))
            for o, w, ti, to in enc:
                occ.append(o)
                wts.append(w)
                terms += ti
                offs += to
                tptr.append(len(terms))
            q_ptr.append(len(occ))
        if n == 0 or not occ:
            return scores, rows
        cache = pg_search.tf_cache(self.total_live, n)
        arr = [np.asarray(q_ptr, np.int32), np.asarray(occ, np.int32), np.asarray(wts, np.float32),
               np.asarray(tptr, np.int32), np.asarray(terms, np.int32), np.asarray(offs, np.int32),
               np.ascontiguousarray(cache, np.float32)]
        with self.torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_pgbm25_search_host(self._h, nq, *[_ptr(a) for a in arr], k, _ptr(scores),
                                                         _ptr(rows), _lib.stream_ptr()), "rmu_pgbm25_search_host")
        return scores, rows


class PgTable:
    """The reference's ``id SERIAL PRIMARY KEY, hash char(32) UNIQUE, content TEXT, metadata TEXT`` on the host.
    Rows are numbered in insertion order; ``on_insert(row, content)`` / ``on_delete(row, content)`` keep an index in
    step.  With ``storage_dir`` every change is one segment file there and the table is replayed from them."""

    def __init__(self, storage_dir: Optional[str] = None, on_insert=None, on_delete=None):
        self.next_id = 1                                  # SERIAL: the next value nextval() hands out
        self.ids: List[int] = []
        self.hashes: List[str] = []
        self.contents: List[str] = []
        self.metas: List[str] = []
        self.alive: List[bool] = []
        self._row_of_hash: Dict[str, int] = {}
        self._row_of_id: Dict[int, int] = {}
        self._on_insert, self._on_delete = on_insert, on_delete
        self._storage_dir = storage_dir
        self._segments = 0
        self._segw: Optional[SegmentWriter] = None
        if storage_dir is not None:
            self._segw = SegmentWriter(self._write_segment)
            self._load()

    def __len__(self) -> int:
        return len(self._row_of_hash)

    def insert(self, documents: Sequence[Any], ids: Sequence[Any]) -> None:
        """``INSERT INTO t (hash, content, metadata) VALUES ... ON CONFLICT (hash) DO NOTHING``, row by row; the whole
        call is refused before anything is stored when a value cannot be stored"""
        recs = []
        for doc, h in zip(documents, ids):
            key = str(h)
            if len(key) > HASH_CHARS:
                raise ValueError(f"value too long for type character({HASH_CHARS}): {key!r}")
            content = doc.page_content
            if "\x00" in content:
                raise ValueError("A string literal cannot contain NUL (0x00) characters.")
            recs.append((key.rstrip(" "), content, json.dumps(doc.metadata)))    # char(n) ignores trailing blanks
        rows = []
        taken = set()                                     # hashes inserted earlier in this call
        for key, content, meta in recs:
            sid = self.next_id                            # nextval() runs before the conflict check
            self.next_id += 1
            if key in self._row_of_hash or key in taken:
                continue
            taken.add(key)
            rows.append([sid, key, content, meta])
        self._apply_rows(rows)
        self._persist({"rows": rows, "next_id": self.next_id})

    def _apply_rows(self, rows) -> None:
        for sid, key, content, meta in rows:
            r = len(self.ids)
            self.ids.append(int(sid))
            self.hashes.append(key)
            self.contents.append(content)
            self.metas.append(meta)
            self.alive.append(True)
            self._row_of_hash[key] = r
            self._row_of_id[int(sid)] = r
            if self._on_insert is not None:
                self._on_insert(r, content)

    def delete(self, ids: Sequence[Any]) -> None:
        """``DELETE FROM t WHERE id IN (...)``; unknown ids delete nothing, an empty list is an SQL error"""
        if len(ids) == 0:
            raise ValueError('syntax error at or near ")": DELETE ... WHERE id IN () needs at least one id')
        want = [int(i) for i in ids]
        gone = self._apply_delete(want)
        if gone:
            self._persist({"deleted": gone})

    def _apply_delete(self, want: Sequence[int]) -> List[int]:
        gone = []
        for sid in want:
            r = self._row_of_id.pop(sid, None)
            if r is None:
                continue
            self.alive[r] = False
            del self._row_of_hash[self.hashes[r]]         # the hash is free again
            gone.append(sid)
            if self._on_delete is not None:
                self._on_delete(r, self.contents[r])
        return gone

    def document(self, row: int, score: float) -> Document:
        meta = {**json.loads(self.metas[row]), "id": self.ids[row], "relevance_score": score}
        return Document(page_content=self.contents[row], metadata=meta)

    # ---------------------------------------------------------------------------------------------- persistence
    def _persist(self, record: Dict[str, Any]) -> None:
        if self._segw is None:
            return
        seg = self._segments
        self._segments += 1
        self._segw.submit(seg, record)

    def _write_segment(self, seg: int, record: Dict[str, Any]) -> None:
        os.makedirs(self._storage_dir, exist_ok=True)
        atomic_savez(os.path.join(self._storage_dir, f"rows_{seg:08d}.npz"),
                     table=np.frombuffer(json.dumps(record).encode(), dtype=np.uint8))

    def _load(self) -> None:
        files = [f for f in sorted(glob.glob(os.path.join(self._storage_dir, "rows_*.npz"))) if not f.endswith(".tmp.npz")]
        for f in files:
            rec = json.loads(bytes(np.load(f, allow_pickle=False)["table"]).decode())
            if "rows" in rec:
                self._apply_rows(rec["rows"])
                self.next_id = max(self.next_id, int(rec["next_id"]))
            else:
                self._apply_delete(rec["deleted"])
        self._segments = len(files)

    def flush(self) -> None:
        if self._segw is not None:
            self._segw.flush()


_warned_memory_only = False


class PostgresBM25Retriever(_Retriever):
    """``server/PostgresBM25Retriever.py`` without Postgres: same constructor keywords, fields, ``add_documents`` /
    ``_get_relevant_documents`` / ``delete`` / ``close`` and return values; BM25 on the GPU."""

    def __init__(self, connection_uri: Any = None, table_name: str = "sparse_vectors", k: int = 4,
                 device: Optional[int] = None, **_: Any):
        global _warned_memory_only
        self.connection_uri = connection_uri               # kept for the reference's field; nothing connects to it
        self.table_name = table_name
        self.k = int(k)
        self.conn = None
        self.cur = None
        self._lock = threading.RLock()                     # Flask serves requests from several threads
        self._index = PgBM25Index(device)
        root = os.environ.get("RMU_STORE_DIR")
        if not root and not _warned_memory_only:
            print("ragmeup_b200.PostgresBM25Retriever: RMU_STORE_DIR is not set, the table lives in memory only "
                  "(rows are not kept across restarts)", file=sys.stderr)
            _warned_memory_only = True
        self._table = PgTable(os.path.join(root, table_name) if root else None,
                              on_insert=lambda r, text: self._index.add(text),
                              on_delete=lambda r, text: self._index.delete(r, text))

    def add_documents(self, documents: List[Document], ids: Optional[List[str]] = None) -> List[str]:
        if ids is None:
            ids = [str(uuid.uuid4()) for _ in range(len(documents))]
        if len(ids) != len(documents):
            raise ValueError("Number of ids must match number of documents")
        with self._lock:
            self._table.insert(documents, ids)
        return ids

    def _search(self, queries: Sequence[str]) -> List[List[Document]]:
        parsed = [pg_search.parse_query(pg_search.sanitize_query(q, os.getenv("use_re2"), os.getenv("re2_prompt")))
                  for q in queries]
        if self.k < 0:
            raise ValueError("LIMIT must not be negative")
        if self.k == 0:
            return [[] for _ in queries]
        with self._lock:
            scores, rows = self._index.search(parsed, self.k)
            # paradedb.score is a float4: Postgres prints it in its shortest exact form, psycopg2 parses that text
            return [[self._table.document(int(r), float(str(s))) for s, r in zip(sr, rr) if r >= 0]
                    for sr, rr in zip(scores, rows)]

    def _get_relevant_documents(self, query: str, **_: Any) -> List[Document]:
        return self._search([query])[0]

    def batch(self, queries: Sequence[str], config: Any = None, **kwargs: Any) -> List[List[Document]]:
        """several queries in one device call"""
        return self._search(list(queries))

    def delete(self, ids: List[Any]) -> None:
        with self._lock:
            self._table.delete(ids)

    def flush(self) -> None:
        """wait until every change is on disk (with ``RMU_STORE_DIR``)"""
        self._table.flush()

    def close(self) -> None:
        self.flush()
