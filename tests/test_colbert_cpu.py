"""CPU: ColBERT checkpoints for HuggingFaceCrossEncoder.  Snapshot detection and refusals, the query / document
tokenisation against hand-written id lists and against oracle/colbert_ref.py, and the oracle pinned against
tests/golden/colbert.npz (minted from transformers' BertModel)."""
import json
import os
import string

import numpy as np
import pytest
import torch

from oracle import colbert_ref
from ragmeup_b200 import weights as W
from ragmeup_b200.colbert import ColBERTTokenizer
from ragmeup_b200.tokenizer import build_wordpiece, synthetic_vocab

VOCAB = synthetic_vocab(30522)
TOK = build_wordpiece(VOCAB)
CLS, SEP, MASK, PAD, QM, DM, DOT = 101, 102, 103, 0, 1, 2, VOCAB["."]


def _words(n, seed=0):
    """n whole-word vocabulary entries that tokenise to one id each"""
    cand = [w for w in VOCAB if w.isalpha() and len(w) > 3][:400]
    rng = np.random.default_rng(seed)
    return [cand[int(i)] for i in rng.choice(len(cand), n, replace=False)]


# ------------------------------------------------------------------------------------------------------- golden
@pytest.mark.parametrize("preset,seed,scale", [("colbertv2.0", 0, 1.0), ("tiny-colbert", 2, 4.0)])
def test_oracle_matches_transformers_golden(golden_dir, preset, seed, scale):
    g = np.load(os.path.join(golden_dir, "colbert.npz"))
    key = f"colbert_{preset}_{seed}_{scale}"
    cfg, w, lin, spec = W.synthetic_colbert(preset, seed, scale)
    Q = colbert_ref.vectors(w, cfg, lin, torch.from_numpy(g[key + "_qids"]).long(), torch.from_numpy(g[key + "_qmask"]).long())
    D = colbert_ref.vectors(w, cfg, lin, torch.from_numpy(g[key + "_dids"]).long(), torch.from_numpy(g[key + "_dmask"]).long())
    assert np.abs(Q.numpy() - g[key + "_Q"]).max() < 4e-6
    dm = g[key + "_dmask"].astype(bool)
    assert np.abs(D.numpy()[dm] - g[key + "_D"][dm]).max() < 4e-6
    got = np.stack([colbert_ref.colbert_score(Q[i], D, torch.from_numpy(dm)).numpy() for i in range(len(Q))])
    assert np.abs(got - g[key + "_scores"]).max() < 4e-6 * spec.query_maxlen


# --------------------------------------------------------------------------------------------------- tokenisation
def test_query_tokens_by_hand():
    spec = W.ColBERTSpec(query_maxlen=8, doc_maxlen=10)
    t = ColBERTTokenizer(TOK, spec)
    a, b, c = _words(3)
    ia, ib, ic = VOCAB[a], VOCAB[b], VOCAB[c]
    long_q = " ".join(_words(12, 1))
    ids, cu, nk = t.queries([f"{a} {b}", "", long_q, f"{a}, {c}"])
    L = [int(VOCAB[x]) for x in long_q.split()]
    want = [[CLS, QM, ia, ib, SEP, MASK, MASK, MASK],
            [CLS, QM, SEP, MASK, MASK, MASK, MASK, MASK],              # an empty query: [CLS] marker [SEP]
            [CLS, QM] + L[:5] + [SEP],                                  # truncated at query_maxlen, specials included
            [CLS, QM, ia, VOCAB[","], ic, SEP, MASK, MASK]]            # punctuation stays in a query
    assert ids.reshape(4, 8).tolist() == want
    assert cu.tolist() == [0, 8, 16, 24, 32]
    assert nk.tolist() == [5, 3, 8, 6]


def test_doc_tokens_and_skiplist_by_hand():
    spec = W.ColBERTSpec(query_maxlen=8, doc_maxlen=10)
    t = ColBERTTokenizer(TOK, spec)
    a, b = _words(2, 3)
    ia, ib = VOCAB[a], VOCAB[b]
    long_d = " ".join(_words(20, 4))
    ids, cu, keep = t.docs([f"{a}, {b}!", "", long_d])
    L = [int(VOCAB[x]) for x in long_d.split()]
    assert ids.tolist() == [CLS, DM, ia, VOCAB[","], ib, VOCAB["!"], SEP,
                            CLS, DM, SEP,
                            CLS, DM] + L[:7] + [SEP]
    assert cu.tolist() == [0, 7, 10, 20]
    assert keep.tolist() == [1, 1, 1, 0, 1, 0, 1, 1, 1, 1] + [1] * 10
    want = sorted({TOK.encode(ch, add_special_tokens=False).ids[0] for ch in string.punctuation})
    assert t.skiplist.tolist() == want and VOCAB["."] in want and CLS not in want and SEP not in want
    # mask_punctuation = False keeps every token
    t2 = ColBERTTokenizer(TOK, W.ColBERTSpec(query_maxlen=8, doc_maxlen=10, mask_punctuation=False))
    assert t2.docs([f"{a}, {b}!"])[2].tolist() == [1] * 7


def test_tokenisation_matches_oracle():
    rng = np.random.default_rng(5)
    words = _words(200, 6) + list(".,;:!?()-'\"")
    texts = ["", "x", "[MASK] a", "[PAD]"] + [" ".join(rng.choice(words, int(rng.integers(1, 80)))) for _ in range(40)]
    for spec in (W.ColBERTSpec(), W.ColBERTSpec(query_maxlen=8, doc_maxlen=12)):
        t = ColBERTTokenizer(TOK, spec)
        ids, cu, nk = t.queries(texts)
        rid, ram = colbert_ref.tokenize_queries(TOK, spec, texts)
        assert ids.reshape(len(texts), -1).tolist() == rid.tolist()
        assert nk.tolist() == ram.sum(1).tolist()
        assert all(int(ram[i, :n].sum()) == n for i, n in enumerate(nk))    # the keys are a prefix
        ids, cu, keep = t.docs(texts)
        rid, ram, rkeep = colbert_ref.tokenize_docs(TOK, spec, texts)
        for b in range(len(texts)):
            n = int(ram[b].sum())
            assert ids[cu[b]:cu[b + 1]].tolist() == rid[b, :n].tolist()
            assert keep[cu[b]:cu[b + 1]].astype(bool).tolist() == rkeep[b, :n].tolist()


# ---------------------------------------------------------------------------------------------------- snapshots
def _snapshot(path, cfg, w, lin, meta=None, config_extra=None, classifier=False, prefix="bert."):
    from safetensors.numpy import save_file
    os.makedirs(path, exist_ok=True)
    d = {"model_type": "bert", "vocab_size": cfg.vocab_size, "hidden_size": cfg.hidden, "num_hidden_layers": cfg.layers,
         "num_attention_heads": cfg.heads, "intermediate_size": cfg.ffn, "max_position_embeddings": cfg.max_pos,
         "type_vocab_size": cfg.type_vocab, "layer_norm_eps": cfg.ln_eps, **(config_extra or {})}
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(d, f)
    t = {prefix + k: v for k, v in w.items()}
    if lin is not None:
        t["linear.weight"] = lin
    if classifier:
        t["classifier.weight"] = np.zeros((1, cfg.hidden), np.float32)
        t["classifier.bias"] = np.zeros(1, np.float32)
    save_file(t, os.path.join(path, "model.safetensors"))
    if meta is not None:
        with open(os.path.join(path, "artifact.metadata"), "w") as f:
            json.dump(meta, f)
    with open(os.path.join(path, "vocab.txt"), "w") as f:
        f.write("\n".join(sorted(VOCAB, key=VOCAB.get)))
    return str(path)


@pytest.fixture(scope="module")
def tiny():
    return W.synthetic_colbert("tiny-colbert", 1)


def test_snapshot_detection(tmp_path, tiny):
    cfg, w, lin, _ = tiny
    meta = {"query_maxlen": 24, "doc_maxlen": 100, "dim": 128, "query_token_id": "[unused0]",
            "doc_token_id": "[unused1]", "attend_to_mask_tokens": False, "similarity": "cosine", "mask_punctuation": True}
    p = _snapshot(tmp_path / "cb", cfg, w, lin, meta, {"architectures": ["HF_ColBERT"]})
    assert W.is_colbert_snapshot(p)
    c2, w2, l2, spec = W.load_colbert_snapshot(p)
    assert (spec.query_maxlen, spec.doc_maxlen, spec.dim) == (24, 100, 128) and np.array_equal(l2, lin)
    assert all(np.array_equal(w2[k], w[k]) for k in w)
    # no architectures, no metadata: linear.weight without a classifier is enough, and the defaults apply
    p = _snapshot(tmp_path / "plain", cfg, w, lin, prefix="")
    assert W.is_colbert_snapshot(p)
    spec = W.load_colbert_snapshot(p)[3]
    assert (spec.query_maxlen, spec.doc_maxlen, spec.query_token, spec.doc_token) == (32, 220, "[unused0]", "[unused1]")
    found = W.resolve_colbert("plain", cache_folder=str(tmp_path))
    assert found is not None and found[4] == p
    # a cross-encoder (classifier present) and an embedder (no linear) are not ColBERT
    assert not W.is_colbert_snapshot(_snapshot(tmp_path / "ce", cfg, w, lin, classifier=True))
    assert W.resolve_colbert(_snapshot(tmp_path / "emb", cfg, w, None)) is None
    assert W.resolve_colbert("synthetic:tiny") is None and W.resolve_colbert("synthetic:tiny-colbert") is not None


@pytest.mark.parametrize("meta,match", [({"similarity": "l2"}, "similarity"),
                                        ({"attend_to_mask_tokens": True}, "attend_to_mask_tokens"),
                                        ({"dim": 64}, "dim 64")])
def test_snapshot_refusals(tmp_path, tiny, meta, match):
    cfg, w, lin, _ = tiny
    p = _snapshot(tmp_path / "r", cfg, w, lin, meta, {"architectures": ["HF_ColBERT"]})
    with pytest.raises(ValueError, match=match):
        W.load_colbert_snapshot(p)


def test_dim_and_model_type_refusals(tmp_path, tiny):
    cfg, w, lin, _ = tiny
    with pytest.raises(ValueError, match="multiple of 128"):
        W.colbert_spec(None, 200)
    assert W.colbert_spec(None, 96).dim == 96 and W.colbert_spec(None, 256).dim == 256
    p = _snapshot(tmp_path / "rob", cfg, w, lin, None, {"architectures": ["HF_ColBERT"], "model_type": "roberta"})
    with pytest.raises(ValueError, match="BERT only"):
        W.resolve_colbert(p)
    # colbert-xm (XMOD) is refused by the encoder's model_type check, as before
    p = _snapshot(tmp_path / "xm", cfg, w, lin, None, {"architectures": ["HF_ColBERT"], "model_type": "xmod"})
    assert W.resolve_colbert(p) is None
    with pytest.raises(ValueError, match="model_type 'xmod' is not supported"):
        W.resolve_model(p, with_head=True)


def test_oracle_maxsim_skips_dropped_tokens():
    """a dropped token never wins, even when every kept dot product is negative"""
    Q = torch.tensor([[1.0, 0.0]])
    D = torch.tensor([[[-1.0, 0.0], [0.0, 0.0], [-0.5, 0.0]]])
    keep = torch.tensor([[True, False, True]])
    assert float(colbert_ref.colbert_score(Q, D, keep)[0]) == -0.5
    s, _ = colbert_ref.maxsim_fsum(Q.numpy(), [0, 1], D[0].numpy(), [0, 3], keep[0].numpy(), [0], [0])
    assert s[0] == -0.5


def test_c_create_refuses_a_linear_weight_the_split_planes_cannot_hold(tiny):
    """`linear` travels as split fp16 planes like every GEMM weight: rmu_colbert_create refuses |w| >= 65520 on the
    host, before any CUDA call, naming the tensor and the index"""
    import ctypes as C
    from ragmeup_b200 import _lib
    cfg, w, lin, spec = tiny
    arrs = [np.ascontiguousarray(w[n], dtype=np.float32) for n, _ in W.weight_names(cfg, False)]
    ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])

    def create(linear):
        h = C.c_void_p()
        rc = _lib.lib().rmu_colbert_create(C.byref(_lib.bert_config_c(cfg)), ptrs, len(arrs), linear.ctypes.data, spec.dim,
                                           C.byref(h))
        if rc == 0:
            _lib.lib().rmu_colbert_destroy(h)
        return rc

    for v in (7e4, -7e4, 65520.0, np.inf):
        big = lin.copy()
        big.reshape(-1)[37] = v
        assert create(big) == -3, v
        assert "linear weight [37]" in _lib.lib().rmu_last_error().decode()
    ok = lin.copy()
    ok.reshape(-1)[37] = 65519.0
    assert create(ok) in (0, -2)                                       # accepted: without a device the next step fails
