"""ColBERT late-interaction scoring on the GPU encoder (``rmu_colbert_*``).

The reference README names ``colbert-ir/colbertv2.0`` as the accuracy pick for ``rerank_model``; it reaches
``HuggingFaceCrossEncoder``, which dispatches here for a ColBERT checkpoint.  Semantics follow colbert-ai's
``QueryTokenizer`` / ``DocTokenizer`` / ``ColBERT.query`` / ``ColBERT.doc`` / ``colbert_score`` [3P-recall: colbert-ai
0.2.x, not installed here; restated in ``oracle/colbert_ref.py``]:

* a query is ``". " + text`` tokenised with [CLS] / [SEP] and truncated to ``query_maxlen`` tokens, position 1 (the
  ``.``) replaced by the query marker, padded to ``query_maxlen`` with [MASK]; the [MASK] rows are queries but not keys
  (``nkeys`` = the real tokens), and all ``query_maxlen`` vectors are kept;
* a document is ``". " + text`` truncated to ``doc_maxlen`` with position 1 the document marker; tokens whose id is the
  first id of a ``string.punctuation`` character (or the padding id) are dropped from scoring;
* on a SentencePiece vocabulary (XLM-R and X-MOD backbones, colbert-xm) the specials are the tokenizer's own: <s>,
  </s>, <mask> and <pad> (id 1) stand for [CLS], [SEP], [MASK] and [PAD], and a marker token the vocabulary lacks is
  <unk>.  The punctuation skiplist keeps its rule, so with Metaspace pre-tokenisation it can hold "▁" (the first piece
  of a mark the vocabulary has no "▁"-piece for), and a lone "▁" is dropped from documents, as colbert-ai does;
* token vectors are ``normalize(linear(h))``; a pair scores sum over query tokens of the max dot product with the
  document's kept tokens.
"""
from __future__ import annotations

import ctypes as C
import string
from typing import List, Sequence, Tuple

import numpy as np
from tokenizers import Tokenizer

from . import _lib
from .encoder import MAX_TOKENS_PER_CALL, BertEncoder
from .tokenizer import _encode_batch
from .weights import BertConfig, ColBERTSpec, weight_names


class ColBERTTokenizer:
    """A private copy of the tokenizer (never reconfigured after construction, so request threads can share it) and
    ColBERT's query / document rules on top of it."""

    def __init__(self, tok: Tokenizer, spec: ColBERTSpec):
        self.spec = spec
        self._tok = Tokenizer.from_str(tok.to_str())
        self._tok.no_truncation()
        self._tok.no_padding()
        tid = self._tok.token_to_id
        if tid("[CLS]") is not None:
            self.cls, self.sep, self.mask, self.pad = tid("[CLS]"), tid("[SEP]"), tid("[MASK]"), tid("[PAD]")
            self.q_marker, self.d_marker = tid(spec.query_token), tid(spec.doc_token)
            if None in (self.cls, self.sep, self.mask, self.pad, self.q_marker, self.d_marker):
                raise ValueError("ColBERT: the tokenizer lacks [CLS], [SEP], [MASK], [PAD] or a marker token "
                                 f"({spec.query_token}, {spec.doc_token})")
        else:
            # a SentencePiece vocabulary (XLM-R, X-MOD): the tokenizer's own specials; a marker the vocabulary lacks
            # is <unk>, what convert_tokens_to_ids returns for it
            self.cls, self.sep, self.mask, self.pad, unk = tid("<s>"), tid("</s>"), tid("<mask>"), tid("<pad>"), tid("<unk>")
            if None in (self.cls, self.sep, self.mask, self.pad, unk):
                raise ValueError("ColBERT: the tokenizer has neither [CLS], [SEP], [MASK], [PAD] nor <s>, </s>, <mask>, "
                                 "<pad>, <unk>")
            self.q_marker, self.d_marker = (unk if t is None else t for t in (tid(spec.query_token), tid(spec.doc_token)))
        skip = set()
        if spec.mask_punctuation:
            for e in self._tok.encode_batch(list(string.punctuation), add_special_tokens=False):
                if e.ids:
                    skip.add(int(e.ids[0]))
        self.skiplist = np.array(sorted(skip), dtype=np.int32)

    def _bodies(self, texts: Sequence[str], maxlen: int, marker: int) -> List[np.ndarray]:
        """[CLS] ". " + text [SEP] truncated to maxlen tokens (specials included), position 1 = marker"""
        enc = _encode_batch(self._tok, [". " + t for t in texts], add_special_tokens=False)
        out = []
        for e in enc:
            body = np.asarray(e.ids[:maxlen - 2], dtype=np.int32)
            s = np.concatenate([[self.cls], body, [self.sep]]).astype(np.int32)
            s[1] = marker
            out.append(s)
        return out

    def queries(self, texts: Sequence[str]) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """-> (ids [nq * query_maxlen], cu [nq + 1], nkeys [nq]); every query is query_maxlen tokens"""
        L = self.spec.query_maxlen
        seqs = self._bodies(texts, L, self.q_marker)
        nkeys = np.array([len(s) for s in seqs], dtype=np.int32)
        ids = np.full((len(seqs), L), self.mask, dtype=np.int32)
        for i, s in enumerate(seqs):
            ids[i, :len(s)] = s
        ids[ids == self.pad] = self.mask                  # colbert-ai maps the padding id to [MASK] everywhere
        cu = np.arange(len(seqs) + 1, dtype=np.int32) * L
        return ids.ravel(), cu, nkeys

    def docs(self, texts: Sequence[str]) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """-> (ids [T], cu [nd + 1], keep [T] uint8)"""
        seqs = self._bodies(texts, self.spec.doc_maxlen, self.d_marker)
        cu = np.zeros(len(seqs) + 1, dtype=np.int32)
        np.cumsum([len(s) for s in seqs], out=cu[1:])
        ids = np.concatenate(seqs).astype(np.int32) if seqs else np.zeros(0, np.int32)
        keep = (~np.isin(ids, self.skiplist) & (ids != self.pad)).astype(np.uint8)
        assert all(keep[cu[b]:cu[b + 1]].any() for b in range(len(seqs))), "a ColBERT document keeps [CLS] and [SEP]"
        return ids, cu, keep


def _index(texts: Sequence[str]) -> Tuple[List[str], np.ndarray]:
    """distinct texts in first-seen order and the index of each input"""
    pos = {}
    idx = np.fromiter((pos.setdefault(t, len(pos)) for t in texts), dtype=np.int32, count=len(texts))
    return list(pos), idx


class ColBERTScorer:
    """The encoder with ColBERT's projection (``rmu_colbert``) and the score of (query, document) pairs."""

    def __init__(self, cfg: BertConfig, weights, linear: np.ndarray, spec: ColBERTSpec, tok: Tokenizer, device=None):
        torch = _lib.require_cuda()
        self.torch = torch
        self.cfg, self.spec = cfg, spec
        self.tokenizer = ColBERTTokenizer(tok, spec)
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        for L in (spec.query_maxlen, spec.doc_maxlen):
            if L > cfg.max_pos or L < 3:
                raise ValueError(f"ColBERT: a length limit of {L} tokens is outside 3..max_position_embeddings "
                                 f"({cfg.max_pos})")
        arrs = [np.ascontiguousarray(weights[n], dtype=np.float32) for n, _ in weight_names(cfg, False)]
        for a, (n, shape) in zip(arrs, weight_names(cfg, False)):
            if tuple(a.shape) != tuple(shape):
                raise ValueError(f"{n}: expected shape {shape}, got {a.shape}")
        self._linear = np.ascontiguousarray(linear, dtype=np.float32)
        if self._linear.shape != (spec.dim, cfg.hidden):
            raise ValueError(f"linear.weight: expected shape {(spec.dim, cfg.hidden)}, got {self._linear.shape}")
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        cc = _lib.bert_config_c(cfg)
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_colbert_create(C.byref(cc), ptrs, len(arrs), self._linear.ctypes.data, spec.dim,
                                                     C.byref(self._h)), "rmu_colbert_create")

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                _lib.lib().rmu_colbert_destroy(h)
            except Exception:
                pass
            self._h = C.c_void_p()

    def _batches(self, pairs):
        pairs = list(pairs)
        if len(pairs) == 0:
            raise IndexError("score() received no text pairs")
        qs, qi = _index([p[0] for p in pairs])
        ds, di = _index([p[1] for p in pairs])
        return self.tokenizer.queries(qs), self.tokenizer.docs(ds), qi, di

    def score(self, text_pairs: Sequence[Tuple[str, str]]) -> np.ndarray:
        """raw MaxSim scores, float32 [n] (host path: one C call)"""
        (qids, qcu, nk), (dids, dcu, keep), qi, di = self._batches(text_pairs)
        out = np.empty(len(qi), dtype=np.float32)
        with self.torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_colbert_score_host(
                self._h, qids.ctypes.data, qcu.ctypes.data, nk.ctypes.data, len(qcu) - 1, len(qids), dids.ctypes.data,
                dcu.ctypes.data, keep.ctypes.data, len(dcu) - 1, len(dids), qi.ctypes.data, di.ctypes.data, len(qi),
                MAX_TOKENS_PER_CALL, out.ctypes.data, _lib.stream_ptr()), "rmu_colbert_score_host")
        return out

    def _dev(self, a, dtype):
        return self.torch.from_numpy(np.ascontiguousarray(a)).to(device=self.device, dtype=dtype, non_blocking=True)

    def vectors_tensor(self, ids, cu, nkeys=None, keep=None):
        """ragged batch -> CUDA fp32 [T, dim] token vectors (one C call; the caller bounds T)"""
        torch = self.torch
        ids_d, cu_d = self._dev(ids, torch.int32), self._dev(cu, torch.int32)
        nk_d = None if nkeys is None else self._dev(nkeys, torch.int32)
        kp_d = None if keep is None else self._dev(keep, torch.uint8)
        out = torch.empty((ids_d.numel(), self.spec.dim), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_colbert_vectors(
                self._h, ids_d.data_ptr(), cu_d.data_ptr(), None if nk_d is None else nk_d.data_ptr(),
                None if kp_d is None else kp_d.data_ptr(), cu_d.numel() - 1, ids_d.numel(),
                int(np.max(np.diff(cu))), out.data_ptr(), _lib.stream_ptr()), "rmu_colbert_vectors")
        return out

    def maxsim_tensor(self, qv, qcu, dv, dcu, keep, pair_q, pair_d):
        """MaxSim of device token vectors -> CUDA fp32 [n_pairs]"""
        torch = self.torch
        qcu_d, dcu_d = self._dev(qcu, torch.int32), self._dev(dcu, torch.int32)
        kp_d = None if keep is None else self._dev(keep, torch.uint8)
        pq, pd = self._dev(pair_q, torch.int32), self._dev(pair_d, torch.int32)
        out = torch.empty(pq.numel(), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().rmu_colbert_maxsim(
                qv.data_ptr(), qcu_d.data_ptr(), dv.data_ptr(), dcu_d.data_ptr(),
                None if kp_d is None else kp_d.data_ptr(), self.spec.dim, pq.data_ptr(), pd.data_ptr(), pq.numel(),
                out.data_ptr(), _lib.stream_ptr()), "rmu_colbert_maxsim")
        return out

    def score_tensor(self, text_pairs: Sequence[Tuple[str, str]]):
        """the same scores as a CUDA fp32 tensor [n]: the query batch, the documents in runs of at most
        MAX_TOKENS_PER_CALL tokens, then MaxSim, all on the device"""
        torch = self.torch
        (qids, qcu, nk), (dids, dcu, keep), qi, di = self._batches(text_pairs)
        qv = self.vectors_tensor(qids, qcu, nk)
        parts = []
        for s, e in BertEncoder._chunks(dcu, MAX_TOKENS_PER_CALL):
            t0, t1 = int(dcu[s]), int(dcu[e])
            parts.append(self.vectors_tensor(dids[t0:t1], (dcu[s:e + 1] - dcu[s]).astype(np.int32), None, keep[t0:t1]))
        dv = parts[0] if len(parts) == 1 else torch.cat(parts, 0)
        return self.maxsim_tensor(qv, qcu, dv, dcu, keep, qi, di)
