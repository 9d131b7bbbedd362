"""GPU: DeBERTa-v3 cross-encoders (mixedbread-ai/mxbai-rerank-*-v1) on the encoder.  E2 with the disentangled
position terms alone against float64 (every query row and the CLS rows, lengths across the exact buckets and up to 512
tokens); the whole stack against the float64 forward; the CLS-only last layer against the full one; the product's
score / score_tensor against the fp32 oracle and the transformers goldens; chunked calls; and RAGMeUp's MMR retrieval
followed by ScoredCrossEncoderReranker.  Bounds follow test_xlmr_gpu.py (u = 2^-24)."""
import math
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import deberta_ref
from oracle import encoder_kernels_ref as ref
from ragmeup_b200.documents import Document
from ragmeup_b200.weights import PRESETS, DebertaConfig, synthetic_bert_weights

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
C_ATT = 8.0                    # as test_xlmr_gpu.py: |err| <= 8 * 2^-22 * max|V| * (1 + A)
SYL = ["ba", "ce", "di", "fo", "gu", "ha", "je", "ki", "lo", "mu", "na", "pe", "qi", "ro", "su", "ta"]


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def _cfg(preset):
    return DebertaConfig(**asdict(PRESETS[preset][0]))


def _texts(n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    return [" ".join("".join(SYL[j] for j in rng.integers(0, len(SYL), rng.integers(1, 4)))
                     for _ in range(int(rng.integers(lo, hi + 1)))) for _ in range(n)]


def _cidx(S, s=256, max_position=512):
    n = max(S, 1)
    b = np.zeros(2 * n - 1, np.int32)
    _lib().check(_lib().lib().rmu_log_bucket_table(s, max_position, n, b.ctypes.data), "rmu_log_bucket_table")
    return np.clip(s + b, 0, 2 * s - 1).astype(np.int32)


# ------------------------------------------------------------------------------------------------- E2 + terms
@pytest.mark.parametrize("cls", [False, True])
def test_attention_disentangled_matches_float64(cuda, cls):
    """every length of the list in one ragged batch: 1, 2, across 128 (the end of the exact buckets) and 256 (a key
    super-block), up to 512; the position window W reaches 511 relative positions"""
    lens = [1, 2, 127, 128, 129, 200, 257, 512]
    H, heads, s = 768, 12, 256
    rng = np.random.default_rng(5)
    T = sum(lens)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    qs = math.log2(math.e) / math.sqrt(3 * 64)
    x = rng.standard_normal((T, 3 * H)).astype(np.float32)
    x[:, :H] *= 0.6 * qs * 8
    pos = rng.standard_normal((2 * s, 2 * H)).astype(np.float32) * 0.5
    pos[:, :H] *= qs * 8
    qkv = [torch.from_numpy(p).cuda() for p in ref.split_f16(x)]
    pp = [torch.from_numpy(p).cuda() for p in ref.split_f16(pos)]
    B = len(lens)
    S = max(lens)
    cidx = _cidx(S)
    W = int(cidx[-1] - cidx[0] + 1)
    assert W == 511
    cls_q = None
    if cls:
        xq = rng.standard_normal((B, H)).astype(np.float32) * 0.6 * qs * 8
        cls_q = [torch.from_numpy(p).cuda() for p in ref.split_f16(xq)]
    rows = B if cls else T
    ws = torch.zeros((rows + T) * heads * W + 2 * S - 1, dtype=torch.float32, device="cuda")
    ch = torch.full((rows, H), float("nan"), dtype=torch.float16, device="cuda")
    cl = torch.full_like(ch, float("nan"))
    cu_d = torch.from_numpy(cu).cuda()
    rc = _lib().lib().rmu_debug_attention_disentangled(
        _ptr(qkv[0]), _ptr(qkv[1]), _ptr(cls_q[0]) if cls else None, _ptr(cls_q[1]) if cls else None, _ptr(cu_d), B, T,
        H, heads, S, _ptr(pp[0]), _ptr(pp[1]), s, cidx.ctypes.data, _ptr(ws), ws.numel(), _ptr(ch), _ptr(cl),
        _lib().stream_ptr())
    _lib().check(rc, "rmu_debug_attention_disentangled")
    torch.cuda.synchronize()
    got = ch.double() + cl.double()
    j = lambda p: p[0].double() + p[1].double()  # noqa: E731
    # c(i, j) of a sequence of n tokens: cidx at r = i - j
    cidx_of = lambda n: cidx[np.arange(n)[:, None] - np.arange(n)[None, :] + S - 1].astype(np.int64)  # noqa: E731
    want = deberta_ref.disentangled_attention_ref(j(qkv), cu, heads, j(pp), cidx_of, cls_q=j(cls_q) if cls else None)
    vmax = float(j(qkv)[:, 2 * H:].abs().max())
    err = float((got - want).abs().max())
    assert torch.isfinite(got).all()
    # scores of up to ~30 in log2 units: the bound of test_xlmr_gpu.py with 1 + A = 32
    assert err <= C_ATT * 2.0 ** -22 * vmax * 32, (err, vmax)
    # a dropped term is far outside the bound
    assert float((want - deberta_ref.disentangled_attention_ref(j(qkv), cu, heads, torch.zeros_like(j(pp)),
                                                               lambda n: np.zeros((n, n), np.int64),
                                                               cls_q=j(cls_q) if cls else None)).abs().max()) > 100 * err


# ------------------------------------------------------------------------------------------------- whole stack
@pytest.mark.parametrize("preset,seed,scale", [("tiny-deberta", 3, 4.0), ("mxbai-rerank-base-v1", 1, 1.0)])
def test_position_planes_at_split_precision(cuda, preset, seed, scale):
    """the work at create time: R = LN_rel(rel_embeddings) (E3) and PQ' | PK = split((R [Wq; Wk]^T + [bq; bk]) * (col <
    H ? log2(e) / sqrt(3 d) : 1)) (E1's QKV epilogue), every layer, against float64 on the split weights.  The bound is
    the split planes' precision, 16 * 2^-22 * (|R| |W|^T + |b|) per element; planes kept as fp16 alone (2^-11) fail it,
    which the test checks on its own reference."""
    from ragmeup_b200.encoder import BertEncoder
    cfg = _cfg(preset)
    w = synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale)
    enc = BertEncoder(cfg, w, with_head=True)
    H, s = cfg.hidden, cfg.position_buckets
    V = lambda n: ref._f64(w[n]).cuda()  # noqa: E731
    R = ref.layernorm_ref(V("encoder.rel_embeddings.weight"), V("encoder.LayerNorm.weight"), V("encoder.LayerNorm.bias"),
                          cfg.ln_eps)[0]
    qs = torch.ones(2 * H, dtype=torch.float64, device="cuda")
    qs[:H] = math.log2(math.e) / math.sqrt(3 * (H // cfg.heads))
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}.attention.self."
        Wqk = torch.cat([ref.split_weight(w[p + n + ".weight"]).cuda() for n in ("query", "key")])
        bqk = torch.cat([V(p + n + ".bias") for n in ("query", "key")])
        want = (R @ Wqk.t() + bqk) * qs
        A = (R.abs() @ Wqk.abs().t() + bqk.abs()) * qs
        hi = torch.empty((2 * s, 2 * H), dtype=torch.float16, device="cuda")
        lo = torch.empty_like(hi)
        _lib().check(_lib().lib().rmu_debug_encoder_position_planes(enc._h, l, _ptr(hi), _ptr(lo), _lib().stream_ptr()),
                     "rmu_debug_encoder_position_planes")
        torch.cuda.synchronize()
        got = hi.double() + lo.double()
        bound = 16 * 2.0 ** -22 * A
        ratio = float(((got - want).abs() / bound).max())
        print(f"\n{preset} layer {l}: max |err| / bound = {ratio:.3g}")
        assert ratio <= 1.0
        assert float(((want.half().double() - want).abs() / bound).max()) > 10, "fp16 alone must fall outside the bound"


# The rule of test_xlmr_gpu.py / test_encoder_stack_gpu.py: against the float64 forward on the split weights, the GPU's
# max and rms error stay within c x those of the fp32 forward on the same weights (deberta_encoder_forward, one sequence
# at a time) + FLOOR u |ref|.  Measured on an H100: tiny x4 4.9 (hidden rms), tiny 1.4, base 21 (bge-reranker-base's
# XLM-R stack: 23).  PQ' | PK kept as fp16 alone raises tiny x4's hidden ratios to about 61 (max) and 42 (rms) in the
# float64 restatement, so that case has c = 20; at scale 1 the position terms are too small for the rule to see it,
# and test_position_planes_at_split_precision checks the planes directly.
FLOOR = 4.0
STACK = {
    "tiny-deberta x4": ("tiny-deberta", 3, 4.0, [0, 1, 2, 64, 129, 257, 200, 512, 0], 20),
    "tiny-deberta": ("tiny-deberta", 0, 1.0, [1, 9, 127, 130, 300, 512], 90),
    "mxbai-rerank-base-v1": ("mxbai-rerank-base-v1", 1, 1.0, [3, 140, 0, 512, 77], 90),
}


def _fp32_forward(w32, cfg, ids, cu):
    H = cfg.hidden
    hidden, logits = [], []
    with torch.no_grad():
        for b in range(len(cu) - 1):
            if cu[b + 1] == cu[b]:
                logits.append(deberta_ref.classifier_head(w32, torch.zeros((1, 1, H), device="cuda")))
                continue
            I = torch.from_numpy(ids[cu[b]:cu[b + 1]].astype(np.int64))[None]
            h = deberta_ref.deberta_encoder_forward(w32, cfg, I, torch.ones_like(I), device="cuda")
            hidden.append(h[0])
            logits.append(deberta_ref.classifier_head(w32, h))
    return {"hidden": torch.cat(hidden).double(), "logits": torch.cat(logits).double()}


def _head_on_hidden(enc, w, ids, cu, mx):
    """rmu_encoder_hidden -> rmu_debug_split_planes -> rmu_debug_cls_head_act (GELU): the logits the CLS-only last
    layer must equal bit for bit"""
    L = _lib()
    lib = L.lib()
    H, nl, B = enc.cfg.hidden, enc.cfg.num_labels, len(cu) - 1
    h = enc.hidden_tokens(ids, None, cu, mx)
    hi = torch.empty(h.shape, dtype=torch.float16, device="cuda")
    lo = torch.empty_like(hi)
    L.check(lib.rmu_debug_split_planes(h.data_ptr(), h.numel(), hi.data_ptr(), lo.data_ptr(), L.stream_ptr()), "split")
    cu_d = torch.from_numpy(cu).cuda()
    head = {k: torch.from_numpy(w[k]).cuda() for k in ("pooler.dense.weight", "pooler.dense.bias", "classifier.weight",
                                                        "classifier.bias")}
    out = torch.empty((B, nl), dtype=torch.float32, device="cuda")
    L.check(lib.rmu_debug_cls_head_act(hi.data_ptr(), lo.data_ptr(), cu_d.data_ptr(), B, H, nl,
                                       head["pooler.dense.weight"].data_ptr(), head["pooler.dense.bias"].data_ptr(),
                                       head["classifier.weight"].data_ptr(), head["classifier.bias"].data_ptr(), 1,
                                       out.data_ptr(), L.stream_ptr()), "cls_head_act")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("case", list(STACK))
def test_deberta_stack_matches_float64_forward(cuda, case):
    """hidden state and logits against the float64 forward on the split weights, by the c x fp32 rule; the CLS-only
    last layer's logits bit-equal to the GELU head on the full stack's hidden state"""
    from ragmeup_b200.encoder import BertEncoder
    preset, seed, scale, lens, c = STACK[case]
    cfg = _cfg(preset)
    w = synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale)
    enc = BertEncoder(cfg, w, with_head=True)
    wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    w32 = {k: ref.split_weight(v).float() if k.endswith(ref.GEMM_WEIGHTS) else v for k, v in wd.items()}
    rng = np.random.default_rng(seed)
    ids = np.concatenate([np.r_[1, rng.integers(4, cfg.vocab_size - 1, max(n - 1, 0))][:n] for n in lens]).astype(np.int32)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    mx = max(lens)
    got = {"hidden": enc.hidden_tokens(ids, None, cu, mx).double(), "logits": enc.classify_tokens(ids, None, cu, mx)}
    want = deberta_ref.deberta_stack_ref(wd, cfg, ids, cu, "split", device="cuda")
    f32 = _fp32_forward(w32, cfg, ids, cu)
    report, fails = [], []
    for name in ("hidden", "logits"):
        g, w_, f = got[name].double(), want[name], f32[name]
        assert torch.isfinite(g).all(), name
        d, e = (g - w_).abs(), (f - w_).abs()
        gmax, grms, fmax, frms = float(d.max()), float(d.pow(2).mean().sqrt()), float(e.max()), float(e.pow(2).mean().sqrt())
        mag_max, mag_rms = float(w_.abs().max()), float(w_.pow(2).mean().sqrt())
        report.append(f"{name} max {gmax:.3g} / fp32 {fmax:.3g} = {gmax / fmax:.3g}, rms {grms:.3g} / {frms:.3g} = "
                      f"{grms / frms:.3g}")
        if gmax > c * fmax + FLOOR * U * mag_max or grms > c * frms + FLOOR * U * mag_rms:
            fails.append(report[-1])
    print(f"\nDeBERTa stack {case}:\n  " + "\n  ".join(report))
    assert not fails, f"{case}: beyond {c} x fp32's error: " + "; ".join(fails)
    # the CLS-only last layer equals the full one: the logits are the hidden state's, through the GELU head alone
    assert torch.equal(_head_on_hidden(enc, w, ids, cu, mx), got["logits"]), "logits differ from the head on the hidden state"
    assert np.array_equal(enc.classify_host(ids, None, cu), got["logits"].cpu().numpy())


def test_golden_logits(cuda, golden_dir):
    """transformers' DebertaV2ForSequenceClassification logits (tests/golden/deberta.npz) from the encoder"""
    from ragmeup_b200.encoder import BertEncoder
    g = np.load(f"{golden_dir}/deberta.npz")
    for seed, scale in ((0, 1.0), (3, 4.0)):
        key = f"deberta_tiny-deberta_{seed}_{scale}"
        cfg = _cfg("tiny-deberta")
        enc = BertEncoder(cfg, synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale), with_head=True)
        lens = g[key + "_mask"].sum(1).astype(int)
        ids = np.concatenate([g[key + "_ids"][b, :n] for b, n in enumerate(lens)]).astype(np.int32)
        cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
        got = enc.classify_host(ids, None, cu)
        want = g[key + "_logits"]
        assert np.abs(got - want).max() < 2e-3 * max(1.0, float(np.abs(want).max()))
        h = enc.hidden_tokens(ids, None, cu, int(lens.max())).cpu().numpy()
        assert np.abs(h[cu[:-1]] - g[key + "_h_first"]).max() < 5e-3


# ------------------------------------------------------------------------------------------------- product
@pytest.fixture(scope="module")
def reranker():
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.weights import resolve_model
    name = "synthetic:tiny-deberta:2:4.0"
    ce = HuggingFaceCrossEncoder(model_name=name)
    cfg, w, *_ = resolve_model(name, with_head=True)
    return ce, w, cfg


def _copy(tok):
    from tokenizers import Tokenizer
    return Tokenizer.from_str(tok.to_str())


def test_score_matches_cross_encoder_predict(reranker):
    """RAGMeUp's call (1 query, 14 documents of about 130 tokens) and a pair past 512 tokens, against the fp32 oracle"""
    ce, w, cfg = reranker
    assert ce.activation == "sigmoid" and ce.max_length == 512 and not ce._types
    q = _texts(1, 6, 12, 1)[0]
    docs = _texts(13, 60, 120, 2) + _texts(1, 400, 600, 3)
    pairs = [(q, d) for d in docs]
    got = ce.score(pairs)
    want = deberta_ref.cross_encoder_predict(w, cfg, _copy(ce.tokenizer), pairs, max_length=512, device="cuda")
    assert got.dtype == np.float32 and got.shape == (14,)
    assert np.abs(got - want).max() < 1e-3
    t = ce.score_tensor(pairs).cpu().numpy()
    assert np.abs(t - got).max() <= 1e-6


def test_chunked_call_equals_small_calls(cuda):
    """mxbai-rerank-base-v1's own workspace bound (1 GiB of position terms: 21 845 tokens per encoder call): a call of
    more tokens than that runs in several encoder calls and scores each pair as small calls do, bit for bit"""
    from ragmeup_b200.cross_encoder import PIPE_PAIRS, HuggingFaceCrossEncoder
    from ragmeup_b200.encoder import POSITION_WS_BYTES
    ce = HuggingFaceCrossEncoder(model_name="synthetic:mxbai-rerank-base-v1:4")
    cfg = ce.config
    assert ce.client.max_tokens_per_call == ce._max_tokens == 21845
    assert ce._max_tokens * 2 * cfg.heads * 2 * cfg.position_buckets * 4 <= POSITION_WS_BYTES
    pairs = [(q, d) for q in _texts(4, 4, 8, 4) for d in _texts(100, 45, 75, 5)]
    _ids, _typ, cu = ce._pairs([p[0] for p in pairs], [p[1] for p in pairs])
    per_pipe = [int(cu[min(s + PIPE_PAIRS, len(pairs))] - cu[s]) for s in range(0, len(pairs), PIPE_PAIRS)]
    assert max(per_pipe) > ce._max_tokens and int(cu[-1]) > ce._max_tokens, (per_pipe, int(cu[-1]))
    big = ce.score(pairs)
    big_t = ce.score_tensor(pairs).cpu().numpy()
    small = np.concatenate([ce.score(pairs[i:i + 14]) for i in range(0, len(pairs), 14)])
    assert np.array_equal(big, small) and np.abs(big_t - small).max() <= 1e-6


def test_mmr_then_deberta_rerank(reranker):
    """Milvus MMR retrieval, then ScoredCrossEncoderReranker with the DeBERTa reranker"""
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.reranker import ScoredCrossEncoderReranker
    from ragmeup_b200.vectorstore import Milvus
    ce, w, cfg = reranker
    emb = HuggingFaceEmbeddings(model_name="synthetic:tiny")
    docs = _texts(200, 20, 60, 6)
    db = Milvus.from_documents([], emb, drop_old=True, connection_args={"uri": "data.db"}, collection_name="deberta")
    db.add_documents([Document(t, {"id": f"id{i}"}) for i, t in enumerate(docs)], ids=[f"id{i}" for i in range(200)])
    retriever = db.as_retriever(search_type="mmr", search_kwargs={"k": 10})
    rr = ScoredCrossEncoderReranker(model=ce, top_n=3)
    for qtext in _texts(3, 5, 12, 7):
        found = retriever.invoke(qtext)
        assert len(found) == 10
        top = rr.compress_documents(found, qtext)
        pairs = [(qtext, d.page_content) for d in found]
        got = ce.score(pairs)
        order = sorted(range(len(found)), key=lambda i: got[i], reverse=True)[:3]
        assert [d.page_content for d in top] == [found[i].page_content for i in order]
        assert [d.metadata["relevance_score"] for d in top] == [got[i] for i in order]
        s = deberta_ref.cross_encoder_predict(w, cfg, _copy(ce.tokenizer), pairs, device="cuda")
        assert np.abs(got - s).max() < 1e-3
