"""Oracle for the Postgres sparse leg: pg_search's tokenizer, query parser and BM25, by brute force.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  PARITY STATUS: unpinned.  The reference
(``server/PostgresBM25Retriever.py``) delegates to ParadeDB 0.11.1 ``pg_search`` (tantivy 0.22), which is absent
here; every rule below is restated from their published sources [3P-recall], independently of
``ragmeup_b200/pg_search.py`` (only the Unicode property table is shared data):

* tokenizer: runs of Rust ``char::is_alphanumeric`` characters, tokens of >= 255 UTF-8 bytes dropped (their position
  stays used), each character lowercased on its own;
* parser: tantivy ``QueryParser`` on ``content`` with ``conjunction_by_default = false`` (see ``parse``);
* BM25: tantivy ``Bm25Weight`` in numpy float32 — idf = ln(1 + (N - df + 0.5) / (df + 0.5)), weight = sum(idf) *
  (1 + K1), tf / (tf + K1 * (1 - B + B * fieldnorm / avg)) with the fieldnorm rounded down to tantivy's
  ``FIELD_NORMS_TABLE`` and avg = total tokens / N; a document's score is the sum of its matched MUST and SHOULD
  clauses in clause order; ties by ascending row.

No inverted index: ``search`` scans every live document for every clause.
"""
from __future__ import annotations

import bisect
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from ragmeup_b200.pg_search import other_alphabetic_ranges

K1 = np.float32(1.2)
B = np.float32(0.75)
_EXTRA = other_alphabetic_ranges()
_EXTRA_LO = [a for a, _ in _EXTRA]


def is_alnum(ch: str) -> bool:
    if ch.isalnum():
        return True
    c = ord(ch)
    i = bisect.bisect_right(_EXTRA_LO, c) - 1
    return i >= 0 and _EXTRA[i][0] <= c <= _EXTRA[i][1]


def tokenize(text: str) -> Tuple[List[str], List[int]]:
    toks, pos, cur, n = [], [], [], 0
    for ch in text + " ":
        if is_alnum(ch):
            cur.append(ch)
            continue
        if cur:
            raw = "".join(cur)
            if len(raw.encode("utf-8", "surrogatepass")) < 255:
                toks.append("".join(c.lower() for c in raw))
                pos.append(n)
            n += 1
            cur = []
    return toks, pos


def field_norms_table() -> np.ndarray:
    """Lucene SmallFloat.byte4ToInt with 24 free values, as tantivy tabulates it"""
    out = list(range(24))
    for b in range(232):
        mant, exp = b & 7, b >> 3
        out.append(24 + (mant if exp == 0 else (mant + 8) * 2 ** (exp - 1)))
    return np.asarray(out, dtype=np.int64)


TABLE = field_norms_table()


def parse(q: str) -> List[Tuple[int, List[str], List[int]]]:
    """(occur 0 SHOULD / 1 MUST / 2 MUST_NOT, tokens, offsets) per clause; raises ValueError on what is refused"""
    if any(c in q for c in "[]{}^~*\\"):
        raise ValueError("refused construct")
    if q.count('"') % 2:
        raise ValueError("unbalanced quote")
    items: List[Tuple[str, str, bool]] = []
    parts = q.split('"')
    for i, part in enumerate(parts):
        if i % 2:                                          # inside quotes
            prefix = ""
            if items and items[-1][1] == "" and not items[-1][2]:
                prefix = items.pop()[0]
            items.append((prefix, part, True))
            continue
        words = part.split()
        ends_glued = bool(part) and not part[-1].isspace() and i + 1 < len(parts)
        for j, w in enumerate(words):
            if w[0] in "+-" and len(w) > 1:
                items.append((w[0], w[1:], False))
            elif w in ("+", "-") and j == len(words) - 1 and ends_glued:
                items.append((w, "", False))              # a prefix glued to the next phrase
            else:
                items.append(("", w, False))
    ops = {t for p, t, qd in items if not qd and not p and t in ("AND", "OR")}
    if len(ops) > 1:
        raise ValueError("AND mixed with OR")
    out = []
    neg = False
    prev_operand = False
    pending = False
    for p, t, qd in items:
        if not qd and not p and t in ("AND", "OR"):
            if not prev_operand or neg:
                raise ValueError("operator without a left operand")
            prev_operand, pending = False, True
            continue
        if not qd and not p and t == "NOT":
            if neg:
                raise ValueError("NOT NOT")
            neg = True
            continue
        occ = {"+": 1, "-": 2}.get(p, 1 if "AND" in ops else 0)
        if neg:
            occ = 2
        neg, prev_operand, pending = False, True, False
        toks, pos = tokenize(t)
        if toks:
            out.append((occ, toks, [x - pos[0] for x in pos]))
    if neg or pending:
        raise ValueError("operator without a right operand")
    return out


def _idf(df: int, n: int) -> np.float32:
    x = (np.float32(n - df) + np.float32(0.5)) / (np.float32(df) + np.float32(0.5))
    return np.float32(np.log(np.float32(np.float32(1.0) + x)))


def search(docs: Sequence[Optional[str]], clauses, k: int) -> Tuple[np.ndarray, np.ndarray]:
    """docs[i] is the content of row i, None for a deleted row -> (float32 scores, rows) of the top k matches"""
    tok = [tokenize(d) if d is not None else None for d in docs]
    live = [i for i, t in enumerate(tok) if t is not None]
    n = len(live)
    if n == 0:
        return np.zeros(0, np.float32), np.zeros(0, np.int64)
    total = sum(len(tok[i][0]) for i in live)
    avg = np.float32(total) / np.float32(n)
    df: Dict[str, int] = {}
    for i in live:
        for t in set(tok[i][0]):
            df[t] = df.get(t, 0) + 1
    n_must = sum(1 for o, _, _ in clauses if o == 1)
    res = []
    for i in live:
        toks, pos = tok[i]
        at: Dict[str, set] = {}
        for t, p in zip(toks, pos):
            at.setdefault(t, set()).add(p)
        fid = int(np.searchsorted(TABLE, len(toks), side="right") - 1)
        norm = np.float32(K1 * np.float32(np.float32(np.float32(1.0) - B) + np.float32(B * np.float32(TABLE[fid])) / avg))
        score = np.float32(0.0)
        musts = 0
        should = False
        excluded = False
        for occ, ts, offs in clauses:
            if any(t not in at for t in ts):
                continue
            tf = sum(1 for p in at[ts[0]] if all(p - offs[0] + o in at[t] for t, o in zip(ts[1:], offs[1:])))
            if tf == 0:
                continue
            if occ == 2:
                excluded = True
                continue
            s = np.float32(0.0)
            for t in ts:
                s = np.float32(s + _idf(df[t], n))
            w = np.float32(s * np.float32(np.float32(1.0) + K1))
            tff = np.float32(tf)
            score = np.float32(score + np.float32(w * np.float32(tff / np.float32(tff + norm))))
            musts += occ == 1
            should |= occ == 0
        if not excluded and musts == n_must and (n_must > 0 or should):
            res.append((score, i))
    res.sort(key=lambda si: (-float(si[0]), si[1]))
    res = res[:k]
    return np.asarray([s for s, _ in res], np.float32), np.asarray([i for _, i in res], np.int64)
