"""PostgresBM25Retriever without a GPU: pg_search rules, the host table, install() and the golden fixture."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import pg_bm25_ref
from ragmeup_b200 import pg_search
from ragmeup_b200.documents import Document
from ragmeup_b200.pg_bm25 import PgTable

import make_golden_pg_bm25


# ------------------------------------------------------------------------------------------------ tokenizer
@pytest.mark.parametrize("text, toks, pos", [
    ("Hello, World! (test) a:b it's", ["hello", "world", "test", "a", "b", "it", "s"], [0, 1, 2, 3, 4, 5, 6]),
    ("state-of-the-art", ["state", "of", "the", "art"], [0, 1, 2, 3]),
    ("U.S. 3.5 v2.0.1", ["u", "s", "3", "5", "v2", "0", "1"], [0, 1, 2, 3, 4, 5, 6]),
    ("Café NAÏVE Ærø", ["café", "naïve", "ærø"], [0, 1, 2]),
    ("東京タワー 北京", ["東京タワー", "北京"], [0, 1]),
    ("ΣΟΦΟΣ ὈΔΥΣΣΕΎΣ", ["σοφοσ", "ὀδυσσεύσ"], [0, 1]),        # no final-sigma rule
    ("under_score a_b", ["under", "score", "a", "b"], [0, 1, 2, 3]),
    ("", [], []),
    ("?! -- ...", [], []),
])
def test_tokenizer_cases(text, toks, pos):
    assert pg_search.tokenize(text) == (toks, pos)


def test_tokenizer_combining_marks_follow_rust():
    # U+093F DEVANAGARI VOWEL SIGN I is Other_Alphabetic: alphanumeric in Rust, not in str.isalnum
    assert not "ि".isalnum()
    assert pg_search.tokenize("कि हिंदी") == (["कि", "हिंदी"], [0, 1])
    # U+0301 COMBINING ACUTE is not alphabetic in either: it splits the token
    assert pg_search.tokenize("ét") == (["e", "t"], [0, 1])
    # circled letters are Other_Alphabetic symbols
    assert pg_search.tokenize("ⓐⓑ") == (["ⓐⓑ"], [0])


def test_tokenizer_drops_long_tokens_and_keeps_their_position():
    assert pg_search.tokenize("a " + "x" * 254 + " b") == (["a", "x" * 254, "b"], [0, 1, 2])
    assert pg_search.tokenize("a " + "x" * 255 + " b") == (["a", "b"], [0, 2])
    assert pg_search.tokenize("é" * 127) == (["é" * 127], [0])              # 254 bytes
    assert pg_search.tokenize("é" * 128) == ([], [])                        # 256 bytes
    assert pg_search.tokenize("a " + "X" * 300 + " b") == pg_bm25_ref.tokenize("a " + "X" * 300 + " b")


# ------------------------------------------------------------------------------------------------ parser
def _p(q):
    return [(c.occur, c.tokens, c.offsets) for c in pg_search.parse_query(q)]


S, M, N = pg_search.SHOULD, pg_search.MUST, pg_search.MUST_NOT


@pytest.mark.parametrize("q, want", [
    ("a b", [(S, ["a"], [0]), (S, ["b"], [0])]),
    ("+a -b c", [(M, ["a"], [0]), (N, ["b"], [0]), (S, ["c"], [0])]),
    ('"new york" city', [(S, ["new", "york"], [0, 1]), (S, ["city"], [0])]),
    ('+"new york" -"los angeles"', [(M, ["new", "york"], [0, 1]), (N, ["los", "angeles"], [0, 1])]),
    ("state-of-the-art", [(S, ["state", "of", "the", "art"], [0, 1, 2, 3])]),
    ("U.S. 3.5", [(S, ["u", "s"], [0, 1]), (S, ["3", "5"], [0, 1])]),
    ("what ? is", [(S, ["what"], [0]), (S, ["is"], [0])]),
    ("a a b", [(S, ["a"], [0]), (S, ["a"], [0]), (S, ["b"], [0])]),
    ("a AND b", [(M, ["a"], [0]), (M, ["b"], [0])]),
    ("a AND -b", [(M, ["a"], [0]), (N, ["b"], [0])]),
    ("a OR b", [(S, ["a"], [0]), (S, ["b"], [0])]),
    ("NOT a b", [(N, ["a"], [0]), (S, ["b"], [0])]),
    ("a and or not", [(S, ["a"], [0]), (S, ["and"], [0]), (S, ["or"], [0]), (S, ["not"], [0])]),
    ('"a ' + "x" * 300 + ' b"', [(S, ["a", "b"], [0, 2])]),
    ('""', []),
    ("", []),
])
def test_parser(q, want):
    assert _p(q) == want
    assert pg_bm25_ref.parse(q) == want


@pytest.mark.parametrize("q, what", [
    ("[a TO b]", "range"), ("{a TO b}", "range"), ("a^2", "boost"), ('"a b"~2', "slop"), ("a~1", "fuzzy"),
    ("a*", "wildcard"), ("a\\-b", "escape"), ('"a b', "unbalanced"), ("a AND b OR c", "AND mixed with OR"),
    ("AND a", "operand"), ("a OR", "operand"), ("NOT", "operand"), ("NOT NOT a", "NOT NOT"),
])
def test_parser_refusals(q, what):
    with pytest.raises(ValueError, match=what):
        pg_search.parse_query(q)
    with pytest.raises(ValueError):
        pg_bm25_ref.parse(q)


def test_sanitize_and_re2(monkeypatch):
    assert pg_search.sanitize_query("(what's) a:b", None, None) == "whats ab"
    q = "what is x\nRead the question again: what is x"
    assert pg_search.sanitize_query(q, "True", "Read the question again:") == "what is x"
    # prompt not found: find() is -1, so the last character goes
    assert pg_search.sanitize_query("what is xy", "True", "Read again:") == "what is x"
    assert pg_search.sanitize_query("what is xy", "False", "Read again:") == "what is xy"
    # unset re2_prompt formats as "None", as the reference's f-string does
    assert pg_search.sanitize_query("a\nNone b", "True", None) == "a"


# ------------------------------------------------------------------------------------------------ arithmetic
def test_field_norms_table():
    t = pg_search.FIELD_NORMS_TABLE
    assert list(t[:41]) == list(range(41)) and t[41] == 42 and t[255] == 2_013_265_944
    assert np.all(np.diff(t) > 0)
    assert list(pg_search.fieldnorm_id([0, 39, 41, 42, 43, 100, 10 ** 9])) == [0, 39, 40, 41, 41, 57, 246]


def test_hand_computed_score():
    docs = ["a b a", "b c", "c d e f"]
    s, r = pg_bm25_ref.search(docs, pg_bm25_ref.parse("a"), 5)
    # N = 3, df(a) = 1, avg = 9 / 3 = 3, doc 0: tf 2, length 3
    idf = np.float32(np.log(np.float32(1) + (np.float32(2.5) / np.float32(1.5))))
    w = np.float32(idf * np.float32(2.2))
    norm = np.float32(np.float32(1.2) * np.float32(np.float32(0.25) + np.float32(np.float32(0.75) * np.float32(3)) / np.float32(3)))
    want = np.float32(w * np.float32(np.float32(2) / np.float32(np.float32(2) + norm)))
    assert list(r) == [0] and s[0] == want
    assert abs(float(want) - 2.2 * np.log(1 + 2.5 / 1.5) * 2 / (2 + 1.2)) < 1e-6
    cache = pg_search.tf_cache(9, 3)
    assert cache[3] == norm
    assert pg_search.clause_weight(pg_search.idf([1], 3)) == w


def test_oracle_matching_rules():
    docs = ["a b", "a c", "b c", "a b c"]
    rows = lambda q: sorted(pg_bm25_ref.search(docs, pg_bm25_ref.parse(q), 10)[1].tolist())
    assert rows("+a b") == [0, 1, 3]
    assert rows("a -c") == [0]
    assert rows("-a") == []
    assert rows("a AND b") == [0, 3]
    assert rows('"a b"') == [0, 3]
    assert rows('"b a"') == []


# ------------------------------------------------------------------------------------------------ the table
def _docs(n, start=0):
    return [Document(page_content=f"text {i}", metadata={"id": f"h{i}", "n": i}) for i in range(start, start + n)]


def test_serial_gaps_and_duplicate_hashes():
    t = PgTable()
    t.insert(_docs(2), ["h0", "h1"])
    t.insert(_docs(3), ["h0", "h2", "h2"])          # h0 conflicts; the second h2 conflicts inside the call
    assert t.ids == [1, 2, 4] and t.next_id == 6
    assert t.contents == ["text 0", "text 1", "text 1"]
    t.delete([4, 99])
    t.insert(_docs(1), ["h2"])                        # the hash is free again after the delete
    assert t.ids[-1] == 6 and len(t) == 3


def test_char32_refusal_and_uuid_default():
    t = PgTable()
    with pytest.raises(ValueError, match="character\\(32\\)"):
        t.insert(_docs(2), ["ok", "x" * 33])
    assert len(t) == 0 and t.next_id == 1
    t.insert(_docs(1), ["x" * 32])
    assert t.ids == [1]
    import uuid
    with pytest.raises(ValueError):
        t.insert(_docs(1), [str(uuid.uuid4())])          # 36 characters, as in the reference
    with pytest.raises(ValueError, match="NUL"):
        t.insert([Document(page_content="a\x00b")], ["n"])


def test_metadata_json_round_trip_and_type_error():
    t = PgTable()
    meta = {"source": "a.pdf", "page": 3, "tags": ["x", "y"], "nested": {"k": 1.5}, "none": None}
    t.insert([Document(page_content="c", metadata=meta)], ["m"])
    assert t.metas[0] == json.dumps(meta)
    d = t.document(0, 1.25)
    assert d.metadata == {**meta, "id": 1, "relevance_score": 1.25}
    with pytest.raises(TypeError):
        t.insert([Document(page_content="a", metadata={}), Document(page_content="b", metadata={"s": {1, 2}})], ["p", "q"])
    assert len(t) == 1 and t.next_id == 2


def test_serial_id_overrides_metadata_id():
    t = PgTable()
    t.insert(_docs(1), ["h0"])
    assert t.document(0, 0.5).metadata["id"] == 1


def test_delete_empty_list_is_refused():
    t = PgTable()
    with pytest.raises(ValueError):
        t.delete([])


def test_table_persistence(tmp_path, monkeypatch):
    monkeypatch.setenv("RMU_STORE_SYNC", "1")
    d = str(tmp_path / "sparse_vectors")
    a = PgTable(d)
    a.insert(_docs(3), ["h0", "h1", "h0"])
    a.delete([2])
    b = PgTable(d)
    assert (b.ids, b.contents, b.alive, b.next_id) == (a.ids, a.contents, a.alive, a.next_id) == ([1, 2], ["text 0", "text 1"], [True, False], 4)
    b.insert(_docs(1), ["h1"])
    assert b.ids[-1] == 4


# ------------------------------------------------------------------------------------------------ install / CUDA
def test_install_registers_module_without_psycopg2():
    code = ("import sys; sys.modules['psycopg2'] = None\n"
            "from ragmeup_b200 import install; install.install()\n"
            "from PostgresBM25Retriever import PostgresBM25Retriever\n"
            "from ragmeup_b200.pg_bm25 import PostgresBM25Retriever as P\n"
            "assert PostgresBM25Retriever is P or PostgresBM25Retriever.__name__ == 'PostgresBM25Retriever'\n")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_pg_bm25_retriever_needs_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from ragmeup_b200 import _lib
    from ragmeup_b200.pg_bm25 import PostgresBM25Retriever
    with pytest.raises(_lib.RmuError):
        PostgresBM25Retriever(connection_uri="postgresql://x", table_name="sparse_vectors", k=4)


# ------------------------------------------------------------------------------------------------ golden
def test_golden_fixture_matches_oracle(golden_dir):
    z = np.load(os.path.join(golden_dir, "pg_bm25.npz"))
    docs = json.loads(bytes(z["docs"]).decode())
    queries = json.loads(bytes(z["queries"]).decode())
    assert docs == make_golden_pg_bm25.corpus() and queries == make_golden_pg_bm25.QUERIES
    live = [None if i in set(z["deleted"].tolist()) else d for i, d in enumerate(docs)]
    k = int(z["k"])
    for q, text in enumerate(queries):
        s, r = pg_bm25_ref.search(live, pg_bm25_ref.parse(text), k)
        assert np.array_equal(z["rows"][q, :len(r)], r) and (z["rows"][q, len(r):] == -1).all()
        assert np.array_equal(z["scores"][q, :len(s)], s)
