"""The pg_search rules behind ``PostgresBM25Retriever``: tokenizer, query parser and BM25 arithmetic.

The reference's sparse leg for ``vector_store=postgres`` (``server/PostgresBM25Retriever.py``) runs
``content @@@ '<query>'`` against a ParadeDB ``pg_search`` BM25 index (ParadeDB 0.11.1, built on tantivy 0.22)
and orders by ``paradedb.score``.  Neither can run here, so every rule in this module is restated from their
published sources and marked **[3P-recall]**; parity with a live ParadeDB is unverified.  This module is the one
place the rules live: ``pg_bm25.py`` (the device index) and ``csrc/rmu_pgbm25.cu`` (the kernel) only follow them.

* Tokenizer [3P-recall]: pg_search's ``default`` tokenizer is tantivy's ``SimpleTokenizer`` -> ``RemoveLongFilter``
  (255 bytes) -> ``LowerCaser``.  A token is a maximal run of characters for which Rust's ``char::is_alphanumeric``
  holds; a token of 255 UTF-8 bytes or more (measured before lowercasing) is dropped but keeps its position, so a
  phrase never matches across it; every character is lowercased on its own (Rust ``char::to_lowercase``: no
  final-sigma rule).  Positions are 0-based token indices.  Rust's predicate is Unicode ``Alphabetic`` or ``Numeric``;
  Python's ``str.isalnum`` misses the ``Other_Alphabetic`` combining marks and symbols, which ``_OTHER_ALPHABETIC``
  adds back (Unicode 15.0, the version of this interpreter's ``unicodedata``).
* Query parser [3P-recall]: tantivy's ``QueryParser`` on the default field ``content`` with
  ``conjunction_by_default = false``, restricted to what survives the reference's ``re.sub(r"[\\(\\):']", "", q)``:
  bare literals SHOULD, ``+lit`` MUST, ``-lit`` MUST_NOT, ``"..."`` phrases, ``AND`` / ``OR`` / ``NOT``.  A literal
  that tokenizes to several tokens is a phrase, one that tokenizes to none is dropped; repeated terms stay separate
  clauses.  Ranges, boosts, slop / fuzzy, wildcards, escapes, an unbalanced quote and AND mixed with OR are refused
  with a ``ValueError`` naming the construct.
* BM25 [3P-recall]: tantivy's ``Bm25Weight`` in float32 with K1 = 1.2, B = 0.75; document lengths through the
  one-byte ``fieldnorm`` code (``FIELD_NORMS_TABLE``).
"""
from __future__ import annotations

import re
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np

# ------------------------------------------------------------------------------------------------ tokenizer
# Characters with Unicode's Alphabetic property that str.isalnum() rejects (Other_Alphabetic: Mn / Mc marks and the
# circled / squared letters), code point ranges in hex, Unicode 15.0.
_OTHER_ALPHABETIC = (
    "345 363-36F 5B0-5BD 5BF 5C1-5C2 5C4-5C5 5C7 610-61A 64B-657 659-65F 670 6D6-6DC 6E1-6E4 6E7-6E8 6ED 711 730-73F "
    "7A6-7B0 816-817 81B-823 825-827 829-82C 8D4-8DF 8E3-8E9 8F0-903 93A-93B 93E-94C 94E-94F 955-957 962-963 981-983 "
    "9BE-9C4 9C7-9C8 9CB-9CC 9D7 9E2-9E3 A01-A03 A3E-A42 A47-A48 A4B-A4C A51 A70-A71 A75 A81-A83 ABE-AC5 AC7-AC9 ACB-ACC "
    "AE2-AE3 AFA-AFC B01-B03 B3E-B44 B47-B48 B4B-B4C B56-B57 B62-B63 B82 BBE-BC2 BC6-BC8 BCA-BCC BD7 C00-C04 C3E-C44 "
    "C46-C48 C4A-C4C C55-C56 C62-C63 C81-C83 CBE-CC4 CC6-CC8 CCA-CCC CD5-CD6 CE2-CE3 CF3 D00-D03 D3E-D44 D46-D48 D4A-D4C "
    "D57 D62-D63 D81-D83 DCF-DD4 DD6 DD8-DDF DF2-DF3 E31 E34-E3A E4D EB1 EB4-EB9 EBB-EBC ECD F71-F83 F8D-F97 F99-FBC "
    "102B-1036 1038 103B-103E 1056-1059 105E-1060 1062-1064 1067-106D 1071-1074 1082-108D 108F 109A-109D 1712-1713 "
    "1732-1733 1752-1753 1772-1773 17B6-17C8 1885-1886 18A9 1920-192B 1930-1938 1A17-1A1B 1A55-1A5E 1A61-1A74 1ABF-1AC0 "
    "1ACC-1ACE 1B00-1B04 1B35-1B43 1B80-1B82 1BA1-1BA9 1BAC-1BAD 1BE7-1BF1 1C24-1C36 1DD3-1DF4 24B6-24E9 2DE0-2DFF "
    "A674-A67B A69E-A69F A802 A80B A823-A827 A880-A881 A8B4-A8C3 A8C5 A8FF A926-A92A A947-A952 A980-A983 A9B4-A9BF A9E5 "
    "AA29-AA36 AA43 AA4C-AA4D AA7B-AA7D AAB0 AAB2-AAB4 AAB7-AAB8 AABE AAEB-AAEF AAF5 ABE3-ABEA FB1E 10376-1037A "
    "10A01-10A03 10A05-10A06 10A0C-10A0F 10D24-10D27 10EAB-10EAC 11000-11002 11038-11045 11073-11074 11080-11082 "
    "110B0-110B8 110C2 11100-11102 11127-11132 11145-11146 11180-11182 111B3-111BF 111CE-111CF 1122C-11234 11237 1123E "
    "11241 112DF-112E8 11300-11303 1133E-11344 11347-11348 1134B-1134C 11357 11362-11363 11435-11441 11443-11445 "
    "114B0-114C1 115AF-115B5 115B8-115BE 115DC-115DD 11630-1163E 11640 116AB-116B5 1171D-1172A 1182C-11838 11930-11935 "
    "11937-11938 1193B-1193C 11940 11942 119D1-119D7 119DA-119DF 119E4 11A01-11A0A 11A35-11A39 11A3B-11A3E 11A51-11A5B "
    "11A8A-11A97 11C2F-11C36 11C38-11C3E 11C92-11CA7 11CA9-11CB6 11D31-11D36 11D3A 11D3C-11D3D 11D3F-11D41 11D43 11D47 "
    "11D8A-11D8E 11D90-11D91 11D93-11D96 11EF3-11EF6 11F00-11F01 11F03 11F34-11F3A 11F3E-11F40 16F4F 16F51-16F87 "
    "16F8F-16F92 16FF0-16FF1 1BC9E 1E000-1E006 1E008-1E018 1E01B-1E021 1E023-1E024 1E026-1E02A 1E08F 1E947 1F130-1F149 "
    "1F150-1F169 1F170-1F189"
)


def other_alphabetic_ranges() -> List[Tuple[int, int]]:
    out = []
    for r in _OTHER_ALPHABETIC.split():
        a, _, b = r.partition("-")
        out.append((int(a, 16), int(b or a, 16)))
    return out


def _token_regex() -> "re.Pattern[str]":
    # [^\W_] is exactly str.isalnum() in Python's re; the Other_Alphabetic ranges complete Rust's is_alphanumeric
    extra = "".join(f"\\U{a:08X}-\\U{b:08X}" for a, b in other_alphabetic_ranges())
    return re.compile(f"(?:[^\\W_]|[{extra}])+")


_TOKEN = _token_regex()
MAX_TOKEN_BYTES = 255          # RemoveLongFilter: a token is kept when its UTF-8 length is below this [3P-recall]


def _lower(tok: str) -> str:
    # str.lower() applies Final_Sigma to a word-final capital sigma; Rust lowercases each char on its own
    return "".join(c.lower() for c in tok) if "Σ" in tok else tok.lower()


def tokenize(text: str) -> Tuple[List[str], List[int]]:
    """pg_search ``default`` tokenizer: (tokens, positions) [3P-recall]"""
    toks: List[str] = []
    pos: List[int] = []
    for i, tok in enumerate(_TOKEN.findall(text)):
        if len(tok) * 4 >= MAX_TOKEN_BYTES and len(tok.encode("utf-8", "surrogatepass")) >= MAX_TOKEN_BYTES:
            continue
        toks.append(_lower(tok))
        pos.append(i)
    return toks, pos


# ------------------------------------------------------------------------------------------------ query parser
SHOULD, MUST, MUST_NOT = 0, 1, 2


@dataclass
class Clause:
    """one query clause: a term (one token) or a phrase (tokens at the given position offsets)"""
    occur: int
    tokens: List[str]
    offsets: List[int]


_REFUSED = [("[", "range queries ([ ])"), ("]", "range queries ([ ])"), ("{", "range queries ({ })"),
            ("}", "range queries ({ })"), ("^", "boosts (^)"), ("~", "slop and fuzzy queries (~)"),
            ("*", "wildcards (*)"), ("\\", "escapes (\\)")]


def sanitize_query(query: str, use_re2: Optional[str], re2_prompt: Optional[str]) -> str:
    """the reference's ``_get_relevant_documents`` before the SQL: with ``use_re2 == "True"`` the query is cut at
    ``query.find("\\n" + re2_prompt)`` (-1 when absent, which drops the last character), then ``( ) : '`` go"""
    if use_re2 == "True":
        query = query[:query.find(f"\n{re2_prompt}")]
    return re.sub(r"[\(\):']", "", query)


def _lexemes(q: str) -> List[Tuple[str, str, bool]]:
    """(prefix, text, quoted) per operand or keyword, split on whitespace; quotes group a phrase"""
    out = []
    i, n = 0, len(q)
    while i < n:
        if q[i].isspace():
            i += 1
            continue
        prefix = ""
        if q[i] in "+-" and i + 1 < n and not q[i + 1].isspace():
            prefix = q[i]
            i += 1
        if q[i] == '"':
            j = q.find('"', i + 1)
            if j < 0:
                raise ValueError("pg_search query: an unbalanced '\"' is not supported")
            out.append((prefix, q[i + 1:j], True))
            i = j + 1
            continue
        j = i
        while j < n and not q[j].isspace() and q[j] != '"':
            j += 1
        out.append((prefix, q[i:j], False))
        i = j
    return out


def parse_query(q: str) -> List[Clause]:
    """sanitised query text -> clauses in query order [3P-recall]"""
    for ch, what in _REFUSED:
        if ch in q:
            raise ValueError(f"pg_search query: {what} are not supported")
    lex = _lexemes(q)
    ops = {t for p, t, quoted in lex if not quoted and not p and t in ("AND", "OR")}
    if len(ops) > 1:
        raise ValueError("pg_search query: AND mixed with OR in one query is not supported")
    conj = "AND" in ops
    clauses: List[Clause] = []
    negate = False
    left = False                                # an operand precedes: AND / OR need one on each side
    pending = False                             # AND / OR seen, its right operand not yet
    for prefix, text, quoted in lex:
        kw = not quoted and not prefix and text in ("AND", "OR", "NOT")
        if kw and text in ("AND", "OR"):
            if not left or negate:
                raise ValueError(f"pg_search query: {text} without an operand on its left")
            left, pending = False, True
            continue
        if kw:                                  # NOT
            if negate:
                raise ValueError("pg_search query: NOT NOT is not supported")
            negate = True
            continue
        occur = MUST if prefix == "+" else MUST_NOT if prefix == "-" else (MUST if conj else SHOULD)
        if negate:
            occur = MUST_NOT
        negate, left, pending = False, True, False
        toks, pos = tokenize(text)
        if toks:
            clauses.append(Clause(occur, toks, [p - pos[0] for p in pos]))
    if negate or pending:
        raise ValueError("pg_search query: AND / OR / NOT without an operand on its right")
    return clauses


# ------------------------------------------------------------------------------------------------ BM25 arithmetic
K1 = np.float32(1.2)
B = np.float32(0.75)


def _field_norms_table() -> np.ndarray:
    """tantivy's FIELD_NORMS_TABLE [3P-recall]: ids 0..23 are the length itself, then Lucene's 4-bit SmallFloat
    (8 steps per power of two) offset by 24; id 255 is 2 013 265 944"""
    t = np.zeros(256, dtype=np.int64)
    for i in range(256):
        if i < 24:
            t[i] = i
        else:
            j = i - 24
            bits, shift = j & 7, (j >> 3) - 1
            t[i] = 24 + (bits if shift < 0 else (bits | 8) << shift)
    return t


FIELD_NORMS_TABLE = _field_norms_table()


def fieldnorm_id(lengths) -> np.ndarray:
    """the largest id whose table value is <= the length (uint8)"""
    return (np.searchsorted(FIELD_NORMS_TABLE, np.asarray(lengths, dtype=np.int64), side="right") - 1).astype(np.uint8)


def idf(df, n_docs: int) -> np.ndarray:
    """ln(1 + (N - df + 0.5) / (df + 0.5)) in float32, the integers converted first"""
    df = np.asarray(df, dtype=np.int64)
    x = ((n_docs - df).astype(np.float32) + np.float32(0.5)) / (df.astype(np.float32) + np.float32(0.5))
    return np.log(np.float32(1.0) + x).astype(np.float32)


def tf_cache(total_tokens: int, n_docs: int) -> np.ndarray:
    """K1 * (1 - B + B * FIELD_NORMS_TABLE[id] / avg) for the 256 ids, avg = total / N in float32"""
    avg = np.float32(total_tokens) / np.float32(n_docs)
    fn = FIELD_NORMS_TABLE.astype(np.float32)
    return (K1 * ((np.float32(1.0) - B) + (B * fn) / avg)).astype(np.float32)


def clause_weight(idfs) -> np.float32:
    """(sum of the clause's term idfs, in order) * (1 + K1): one idf for a term, Bm25Weight::for_terms for a phrase"""
    s = np.float32(0.0)
    for v in idfs:
        s = np.float32(s + np.float32(v))
    return np.float32(s * (np.float32(1.0) + K1))
