"""GPU: ColBERT on the encoder.  E2 with a key limit per sequence and MaxSim, each alone against float64; the whole
ColBERT stack (token vectors and scores) against the float64 forward on the split weights; then the product:
HuggingFaceCrossEncoder.score on ColBERT checkpoints against oracle/colbert_ref.py, chunking, threads and RAGMeUp's
rerank retriever.  Bounds follow tests/test_encoder_kernels_gpu.py and tests/test_encoder_stack_gpu.py (u = 2^-24)."""
import functools
import math
import threading

import numpy as np
import pytest
import torch

from oracle import colbert_ref
from oracle import encoder_kernels_ref as ref
from ragmeup_b200.weights import synthetic_colbert

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def _i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


# ------------------------------------------------------------------------------------------------ E2 + key limit
C_ATT = 8.0      # test_encoder_kernels_gpu.py's c_att: the key limit only moves where the key loop stops


def _attention_keys(qkv, cu, nkeys, H, heads, warps):
    T = qkv[0].shape[0]
    ch = torch.full((T, H), float("nan"), dtype=torch.float16, device="cuda")
    cl = torch.full_like(ch, float("nan"))
    cu_d, nk_d = _i32(cu), _i32(nkeys)                  # held: a freed temporary's block could be handed out again
    rc = _lib().lib().rmu_debug_attention_keys(_ptr(qkv[0]), _ptr(qkv[1]), _ptr(cu_d), _ptr(nk_d), len(cu) - 1,
                                               H, heads, int(np.diff(cu).max()), warps, _ptr(ch), _ptr(cl),
                                               _lib().stream_ptr())
    _lib().check(rc, "rmu_debug_attention_keys")
    torch.cuda.synchronize()
    return ch, cl


def _attention_plain(qkv, cu, H, heads, warps):
    T = qkv[0].shape[0]
    ch = torch.full((T, H), float("nan"), dtype=torch.float16, device="cuda")
    cl = torch.full_like(ch, float("nan"))
    cu_d = _i32(cu)
    _lib().check(_lib().lib().rmu_debug_attention(_ptr(qkv[0]), _ptr(qkv[1]), _ptr(cu_d), len(cu) - 1, H, heads,
                                                  int(np.diff(cu).max()), warps, _ptr(ch), _ptr(cl), _lib().stream_ptr()),
                 "rmu_debug_attention")
    torch.cuda.synchronize()
    return ch, cl


# S = 32 with every key count 1..32; long sequences with the limit around the 256-key super-block edge
LENS = [32] * 32 + [300, 300, 300, 600, 600, 257, 512]
NKEYS = list(range(1, 33)) + [255, 256, 257, 256, 500, 1, 511]


@pytest.mark.parametrize("H,heads,warps", [(384, 12, 10), (768, 12, 10)])
def test_key_limited_attention_matches_float64(cuda, H, heads, warps):
    rng = np.random.default_rng(H + warps)
    dh = H // heads
    cu = np.r_[0, np.cumsum(LENS)].astype(np.int64)
    T = int(cu[-1])
    q, k, v = (rng.standard_normal((T, H)) for _ in range(3))
    q *= math.log2(math.e) / math.sqrt(dh)
    for b, n in enumerate(NKEYS):                       # excluded rows hold V = 1e4: any leak is visible at once
        v[cu[b] + n:cu[b + 1]] = 1e4
    qkv = tuple(torch.from_numpy(p).cuda() for p in ref.split_f16(np.concatenate([q, k, v], 1).astype(np.float32)))
    ch, cl = _attention_keys(qkv, cu, NKEYS, H, heads, warps)
    got = ch.double() + cl.double()
    want, A = colbert_ref.attention_keys_ref(qkv[0], qkv[1], cu, NKEYS, heads)
    vv = qkv[0][:, 2 * H:].double() + qkv[1][:, 2 * H:].double()
    worst = 0.0
    for b, n in enumerate(NKEYS):
        t0, t1 = int(cu[b]), int(cu[b + 1])
        vmax = vv[t0:t0 + n].abs().view(n, heads, dh).amax((0, 2))       # over the keys the rows may read
        bound = 2.0 ** -22 * vmax[None, :, None] * (1 + A[t0:t1, :, None])
        worst = max(worst, float(((got[t0:t1] - want[t0:t1]).abs().view(t1 - t0, heads, dh) / bound).max()))
    print(f"\nE2 key limit H={H} warps={warps}: worst |err|/(2^-22 max|V| (1+A)) = {worst:.3g}")
    assert worst <= C_ATT
    # nkeys = S: bit-identical to the kernel without a limit; nkeys past S clamps to S
    full = np.diff(cu).astype(np.int32)
    for nk in (full, full + 7):
        kh, kl = _attention_keys(qkv, cu, nk, H, heads, warps)
        ph, pl = _attention_plain(qkv, cu, H, heads, warps)
        assert _bits_equal(kh, ph) and _bits_equal(kl, pl)


# ------------------------------------------------------------------------------------------------------- MaxSim
def _maxsim(q, qcu, d, dcu, keep, pq, pd):
    out = torch.full((len(pq),), float("nan"), dtype=torch.float32, device="cuda")
    kp = None if keep is None else torch.from_numpy(np.asarray(keep, np.uint8)).cuda()
    qcu_d, dcu_d, pq_d, pd_d = _i32(qcu), _i32(dcu), _i32(pq), _i32(pd)
    _lib().check(_lib().lib().rmu_colbert_maxsim(_ptr(q), _ptr(qcu_d), _ptr(d), _ptr(dcu_d), _ptr(kp), q.shape[1],
                                                 _ptr(pq_d), _ptr(pd_d), len(pq), _ptr(out), _lib().stream_ptr()),
                 "rmu_colbert_maxsim")
    torch.cuda.synchronize()
    return out


def _unit(rng, n, dim):
    x = rng.standard_normal((n, dim))
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def test_maxsim_matches_fsum_replay(cuda):
    rng = np.random.default_rng(3)
    dim, Lq = 128, 32
    q = _unit(rng, 3 * Lq, dim)
    qcu = np.arange(4) * Lq
    lens = [3, 512, 100, 37, 3]
    dcu = np.r_[0, np.cumsum(lens)]
    d = _unit(rng, int(dcu[-1]), dim)
    keep = (rng.random(int(dcu[-1])) > 0.2).astype(np.uint8)
    for b in range(len(lens)):
        keep[dcu[b]] = keep[dcu[b + 1] - 1] = 1
    # document 4: every kept dot with query 0's first token is negative, and the skipped token is a zero vector that
    # would win with 0 if it were a candidate
    t0 = int(dcu[4])
    d[t0], d[t0 + 1], d[t0 + 2] = -q[0], 0.0, -0.5 * q[0]
    keep[t0:t0 + 3] = (1, 0, 1)
    d[dcu[1] + 5] = q[Lq + 7]                           # a skipped exact match in the 512-token document
    keep[dcu[1] + 5] = 0
    pq, pd = np.repeat(np.arange(3), len(lens)), np.tile(np.arange(len(lens)), 3)
    got = _maxsim(torch.from_numpy(q).cuda(), qcu, torch.from_numpy(d).cuda(), dcu, keep, pq, pd).cpu().numpy()
    want, M = colbert_ref.maxsim_fsum(q, qcu, d, dcu, keep, pq, pd)
    ratio = float((np.abs(got - want) / ((dim + Lq) * U * M)).max())
    print(f"\nMaxSim: worst |err| / ((dim + Lq) u M) = {ratio:.3g}")
    assert ratio <= 1.0
    best0 = max(float(np.dot(q[0], d[t0 + j])) for j in (0, 2))
    assert best0 == pytest.approx(-0.5, abs=1e-6)
    # a pair alone equals its score in a batch of 1000, bit for bit
    rng2 = np.random.default_rng(4)
    bq, bd = rng2.integers(0, 3, 1000), rng2.integers(0, len(lens), 1000)
    big = _maxsim(torch.from_numpy(q).cuda(), qcu, torch.from_numpy(d).cuda(), dcu, keep, bq, bd)
    for n in (0, 1, 499, 999):
        alone = _maxsim(torch.from_numpy(q).cuda(), qcu, torch.from_numpy(d).cuda(), dcu, keep, bq[n:n + 1], bd[n:n + 1])
        assert torch.equal(alone[0], big[n])
    flat = np.asarray([got[i * len(lens) + j] for i, j in zip(bq, bd)], np.float32)
    assert np.array_equal(big.cpu().numpy(), flat)


# -------------------------------------------------------------------------------------------------- whole stack
FLOOR = 4.0
# (preset, scale, c): c bounds the max and RMS error ratios to fp32's, twice the worst measured on an H100 (DESIGN.md)
STACK = {"colbertv2.0": ("colbertv2.0", 1.0, 84.0), "tiny-colbert x4": ("tiny-colbert", 4.0, 24.0)}


def _fp32_vectors(w32, cfg, lin32, ids, cu, nkeys):
    lens = np.diff(cu)
    S = int(lens.max())
    I = np.zeros((len(lens), S), np.int64)
    M = np.zeros_like(I)
    for b, n in enumerate(lens):
        I[b, :n] = ids[cu[b]:cu[b + 1]]
        M[b, :nkeys[b]] = 1
    V = colbert_ref.vectors(w32, cfg, lin32, torch.from_numpy(I), torch.from_numpy(M), device="cuda")
    return torch.cat([V[b, :n] for b, n in enumerate(lens)]).double()


@pytest.mark.parametrize("case", list(STACK))
def test_colbert_stack_matches_float64_forward(cuda, case):
    from ragmeup_b200.colbert import ColBERTScorer
    from ragmeup_b200.tokenizer import load_tokenizer
    preset, scale, c = STACK[case]
    cfg, w, lin, spec = synthetic_colbert(preset, 5, scale)
    sc = ColBERTScorer(cfg, w, lin, spec, load_tokenizer(None, cfg.vocab_size))
    rng = np.random.default_rng(8)
    Lq = spec.query_maxlen
    nq = [3, Lq // 2, Lq]
    qids = np.concatenate([np.r_[101, 1, rng.integers(200, cfg.vocab_size, n - 3), 102, [103] * (Lq - n)] for n in nq])
    qcu = np.arange(len(nq) + 1) * Lq
    dl = [3, 17, spec.doc_maxlen, 40]
    dids = np.concatenate([np.r_[101, 2, rng.integers(200, cfg.vocab_size, n - 3), 102] for n in dl])
    dcu = np.r_[0, np.cumsum(dl)]
    keep = (rng.random(len(dids)) > 0.15).astype(np.uint8)
    keep[dcu[:-1]] = 1
    qv = sc.vectors_tensor(qids, qcu, np.asarray(nq, np.int32))
    dv = sc.vectors_tensor(dids, dcu, None, keep)
    torch.cuda.synchronize()
    wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    ld = torch.from_numpy(lin).cuda()
    w32 = {k: ref.split_weight(v).float() if k.endswith(ref.GEMM_WEIGHTS) else v for k, v in wd.items()}
    l32 = ref.split_weight(ld).float()
    want_q = colbert_ref.colbert_stack_ref(wd, cfg, ld, qids, qcu, nq, None, "split", device="cuda")["vectors"]
    want_d = colbert_ref.colbert_stack_ref(wd, cfg, ld, dids, dcu, None, keep, "split", device="cuda")["vectors"]
    f_q = _fp32_vectors(w32, cfg, l32, qids, qcu, nq)
    f_d = _fp32_vectors(w32, cfg, l32, dids, dcu, dl) * torch.from_numpy(keep).cuda()[:, None]
    pq, pd = np.repeat(np.arange(len(nq)), len(dl)), np.tile(np.arange(len(dl)), len(nq))
    kd = torch.from_numpy(keep.astype(bool)).cuda()

    def scores(Q, D):
        out = []
        for a, b in zip(pq, pd):
            s = Q[qcu[a]:qcu[a + 1]] @ D[dcu[b]:dcu[b + 1]].T
            s[:, ~kd[dcu[b]:dcu[b + 1]]] = -math.inf
            out.append(s.max(1).values.sum())
        return torch.stack(out)

    got_s = sc.maxsim_tensor(qv, qcu, dv, dcu, keep, pq, pd).double()
    outs = {"query vectors": (qv.double(), want_q, f_q), "doc vectors": (dv.double(), want_d, f_d),
            "scores": (got_s, scores(want_q, want_d), scores(f_q, f_d))}
    report, fails = [], []
    for name, (g, w_, f) in outs.items():
        assert torch.isfinite(g).all(), name
        d_, e = (g - w_).abs(), (f - w_).abs()
        gmax, grms, fmax, frms = float(d_.max()), float(d_.pow(2).mean().sqrt()), float(e.max()), float(e.pow(2).mean().sqrt())
        mag_max, mag_rms = float(w_.abs().max()), float(w_.pow(2).mean().sqrt())
        report.append(f"{name} max {gmax:.3g} / fp32 {fmax:.3g} = {gmax / fmax:.3g}, rms {grms:.3g} / {frms:.3g} = "
                      f"{grms / frms:.3g}")
        if gmax > c * fmax + FLOOR * U * mag_max or grms > c * frms + FLOOR * U * mag_rms:
            fails.append(report[-1])
    print(f"\nColBERT stack {case}:\n  " + "\n  ".join(report))
    assert (dv[~kd] == 0).all()
    assert not fails, f"{case}: beyond {c} x fp32's error: " + "; ".join(fails)
    # one document alone equals its rows in the batch
    b = 2
    one = sc.vectors_tensor(dids[dcu[b]:dcu[b + 1]], np.array([0, dl[b]], np.int32), None, keep[dcu[b]:dcu[b + 1]])
    assert torch.equal(one, dv[dcu[b]:dcu[b + 1]])


# -------------------------------------------------------------------------------------------------------- product
@pytest.fixture(scope="module")
def scorers(cuda):
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    out = {}
    for name in ("synthetic:colbertv2.0:1", "synthetic:colbertv2.0:1:4", "synthetic:tiny-colbert:2"):
        out[name] = HuggingFaceCrossEncoder(model_name=name)
    return out


@functools.lru_cache(maxsize=1)
def _vocab():
    from ragmeup_b200.tokenizer import synthetic_vocab
    return synthetic_vocab(30522)


def _texts(n, lo, hi, seed):
    from ragmeup_b200.tokenizer import synthetic_sentences
    return synthetic_sentences(_vocab(), n, lo, hi, seed=seed)


def _oracle(ce, name, pairs):
    from ragmeup_b200.tokenizer import load_tokenizer
    parts = name.split(":")
    cfg, w, lin, spec = synthetic_colbert(parts[1], int(parts[2]), float(parts[3]) if len(parts) > 3 else 1.0)
    return colbert_ref.score_pairs(w, cfg, lin, spec, load_tokenizer(None, cfg.vocab_size), pairs, device="cuda")


BOUND = 1e-3


@pytest.mark.parametrize("name", ["synthetic:colbertv2.0:1", "synthetic:colbertv2.0:1:4"])
@pytest.mark.parametrize("shape", ["ragmeup", "bulk", "long"])
def test_score_matches_colbert_oracle(scorers, name, shape):
    ce = scorers[name]
    if shape == "ragmeup":            # one query, 14 documents (RAGMeUp's rerank call)
        q = _texts(1, 5, 12, 1)[0]
        pairs = [(q, d) for d in _texts(14, 60, 120, 2)]
    elif shape == "bulk":             # 100 pairs over several queries, repeated texts
        qs, ds = _texts(5, 3, 40, 3) + ["", "?"], _texts(40, 1, 150, 4) + ["", ". , ;"]
        rng = np.random.default_rng(5)
        pairs = [(qs[int(rng.integers(len(qs)))], ds[int(rng.integers(len(ds)))]) for _ in range(100)]
    else:                             # documents cut at doc_maxlen, queries cut at query_maxlen
        pairs = [(q, d) for q, d in zip(_texts(3, 40, 60, 6), _texts(3, 250, 400, 7))]
    got = ce.score(pairs)
    want = _oracle(ce, name, pairs)
    assert got.dtype == np.float32 and got.shape == (len(pairs),)
    err = float(np.abs(got - want).max())
    print(f"\n{name} {shape}: max |score - oracle| = {err:.3g}")
    assert err <= BOUND
    i, j = np.triu_indices(len(pairs), 1)
    far = np.abs(want[i] - want[j]) > 2 * BOUND
    assert (np.sign(got[i] - got[j])[far] == np.sign(want[i] - want[j])[far]).all()
    t = ce.score_tensor(pairs)
    assert torch.equal(t.cpu(), torch.from_numpy(got))


def test_empty_list_raises(scorers):
    ce = scorers["synthetic:tiny-colbert:2"]
    with pytest.raises(IndexError):
        ce.score([])
    with pytest.raises(IndexError):
        ce.score_tensor([])


def test_a_call_past_the_token_limit_equals_two_calls(scorers):
    from ragmeup_b200.encoder import MAX_TOKENS_PER_CALL
    ce = scorers["synthetic:tiny-colbert:2"]
    L = ce.colbert.spec.doc_maxlen
    n = MAX_TOKENS_PER_CALL // L + 3
    base = _texts(50, 80, 90, 100)
    docs = [f"doc {i} " + base[i % 50] for i in range(n)]
    ids, cu, _ = ce.colbert.tokenizer.docs(docs)
    assert int(cu[-1]) > MAX_TOKENS_PER_CALL
    q = _texts(2, 4, 9, 8)
    pairs = [(q[i % 2], d) for i, d in enumerate(docs)]
    whole = ce.score(pairs)
    h = len(pairs) // 2
    assert np.array_equal(whole, np.concatenate([ce.score(pairs[:h]), ce.score(pairs[h:])]))
    assert torch.equal(ce.score_tensor(pairs).cpu(), torch.from_numpy(whole))


def test_four_threads_on_one_instance_give_the_serial_results(scorers):
    ce = scorers["synthetic:colbertv2.0:1"]
    jobs = [[(q, d) for d in _texts(14, 30, 90, 20 + k)] for k, q in enumerate(_texts(8, 4, 12, 19))]
    serial = [ce.score(j) for j in jobs]
    got = [None] * len(jobs)

    def run(k):
        for _ in range(3):
            got[k] = ce.score(jobs[k])

    th = [threading.Thread(target=run, args=(k,)) for k in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for k in range(4):
        assert np.array_equal(got[k], serial[k])


def test_ragmeup_rerank_retriever_on_a_colbert_snapshot(cuda, tmp_path, monkeypatch):
    """ContextualCompressionRetriever(ScoredCrossEncoderReranker(HuggingFaceCrossEncoder(<ColBERT snapshot>), top_n=3),
    EnsembleRetriever([BM25, Milvus mmr])) as RAGHelper builds it with rerank_model=colbert-ir/colbertv2.0"""
    import json
    import os
    from dataclasses import asdict

    from safetensors.numpy import save_file

    from oracle import bert_ref, flat_ref
    from oracle import hybrid_ref as HR
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.documents import Document
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.reranker import ScoredCrossEncoderReranker
    from ragmeup_b200.retrievers import BM25Retriever, ContextualCompressionRetriever, EnsembleRetriever
    from ragmeup_b200.tokenizer import synthetic_vocab
    from ragmeup_b200.vectorstore import Milvus
    from ragmeup_b200.weights import resolve_model
    cfg, w, lin, spec = synthetic_colbert("colbertv2.0", 3, 4.0)
    snap = tmp_path / "colbert-ir" / "colbertv2.0"
    os.makedirs(snap)
    with open(snap / "config.json", "w") as f:
        json.dump({"architectures": ["HF_ColBERT"], "model_type": "bert", "vocab_size": cfg.vocab_size,
                   "hidden_size": cfg.hidden, "num_hidden_layers": cfg.layers, "num_attention_heads": cfg.heads,
                   "intermediate_size": cfg.ffn, "max_position_embeddings": cfg.max_pos, "type_vocab_size": 2}, f)
    save_file({**{"bert." + k: v for k, v in w.items()}, "linear.weight": lin}, str(snap / "model.safetensors"))
    with open(snap / "artifact.metadata", "w") as f:
        json.dump({"query_maxlen": 32, "doc_maxlen": 180, "dim": 128, "similarity": "cosine",
                   "attend_to_mask_tokens": False, "query_token_id": "[unused0]", "doc_token_id": "[unused1]"}, f)
    vocab = synthetic_vocab(30522)
    with open(snap / "vocab.txt", "w") as f:
        f.write("\n".join(sorted(vocab, key=vocab.get)))
    monkeypatch.setenv("RAGMEUP_MODEL_DIR", str(tmp_path))
    ce = HuggingFaceCrossEncoder(model_name="colbert-ir/colbertv2.0")
    assert ce.colbert is not None and ce.colbert.spec.doc_maxlen == 180
    compressor = ScoredCrossEncoderReranker(model=ce, top_n=3)
    from ragmeup_b200.tokenizer import load_tokenizer
    otok = load_tokenizer(str(snap), cfg.vocab_size)

    emb = HuggingFaceEmbeddings(model_name="synthetic:all-MiniLM-L6-v2:0", model_kwargs={"device": "cuda"})
    texts = _texts(400, 30, 60, 17)
    queries = [" ".join(t.split()[3:9]) for t in texts[5:8]]
    documents = [Document(t, {"source": f"f{i % 5}.txt", "id": f"id{i}"}) for i, t in enumerate(texts)]
    db = Milvus.from_documents([], emb, drop_old=True, connection_args={"uri": "data.db"}, collection_name="cb")
    db.add_documents(documents, ids=[d.metadata["id"] for d in documents])
    sparse = BM25Retriever.from_texts(texts, metadatas=[d.metadata for d in documents])
    dense = db.as_retriever(search_type="mmr", search_kwargs={"k": 10})
    ensemble = EnsembleRetriever(retrievers=[sparse, dense], weights=[0.5, 0.5])
    rerank = ContextualCompressionRetriever(base_compressor=compressor, base_retriever=ensemble)

    ecfg, ew, *_ = resolve_model(emb.model_name, with_head=False)
    ecfg = bert_ref.BertCfg(**asdict(ecfg))
    X = bert_ref.st_encode(ew, ecfg, emb.tokenizer, texts, "mean", True, 256)
    o_sparse = HR.BM25Retriever.from_texts(texts, make_doc=lambda t, m: t)
    for q in queries:
        sp = o_sparse.invoke(q)
        qv = np.asarray(bert_ref.hf_embed_query(ew, ecfg, emb.tokenizer, q, max_seq_length=256), dtype=np.float32)
        de = [texts[r] for r in flat_ref.mmr_search(qv[None], X, 10, "l2", fetch_k=20, lambda_mult=0.5)[0]]
        fused = HR.weighted_reciprocal_rank([sp, de], [0.5, 0.5], key=lambda t: t)
        want = colbert_ref.score_pairs(w, cfg, lin, spec, otok, [(q, t) for t in fused], device="cuda")
        out = rerank.invoke(q)
        assert len(out) == 3
        got = np.array([d.metadata["relevance_score"] for d in out])
        pos = [fused.index(d.page_content) for d in out]
        assert np.abs(got - want[pos]).max() <= BOUND
        order = np.argsort(-want, kind="stable")
        assert all(want[p] >= want[order[2]] - 2 * BOUND for p in pos)       # the oracle's top three, up to near-ties
