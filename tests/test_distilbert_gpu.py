"""DistilBERT checkpoints and sentence-transformers Dense modules on the GPU encoder: the Dense kernel alone against
float64 (rmu_debug_dense), the tiny-distilbert encoder with two Dense chains against tests/golden/distilbert.npz, temp
DistilBERT snapshots through the drop-ins against transformers in float64, and a LaBSE-shaped BERT (CLS, Dense,
Normalize) against the float64 encoder oracle."""
import importlib.util
import os
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import dense_ref, provenance_ref
from oracle import encoder_kernels_ref as ref
from ragmeup_b200.weights import (PRESETS, BertConfig, DistilBertConfig, dense_layers, synthetic_bert_weights,
                                  synthetic_dense_weights)

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
U = 2.0 ** -24


def _golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_distilbert", os.path.join(HERE, "golden",
                                                                                        "make_golden_distilbert.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


G = _golden_module()


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _dense_dev(x, W, b, act, normalize):
    from ragmeup_b200 import _lib
    B, n_in = x.shape
    y = torch.empty((B, W.shape[0]), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().rmu_debug_dense(x.data_ptr(), B, n_in, W.shape[0], W.data_ptr(),
                                          None if b is None else b.data_ptr(), act, int(normalize), y.data_ptr(),
                                          _lib.stream_ptr()), "rmu_debug_dense")
    torch.cuda.synchronize()
    return y


# (n_in, n_out): in = out, in > out, in < out, and widths that are not multiples of 32
WIDTHS = [(128, 128), (768, 512), (768, 500), (128, 1000), (33, 7), (1, 65)]


@pytest.mark.parametrize("n_in,n_out", WIDTHS)
@pytest.mark.parametrize("B", [1, 9, 4096])
def test_dense_kernel_matches_float64(cuda, n_in, n_out, B):
    g = torch.Generator(device="cpu").manual_seed(n_in * 7 + n_out + B)
    x = torch.randn((B, n_in), generator=g).cuda()
    W = (torch.randn((n_out, n_in), generator=g) / n_in ** 0.5).cuda()
    b = (0.1 * torch.randn(n_out, generator=g)).cuda()
    for act in (0, 1):
        for bias in (None, b):
            for normalize in (False, True):
                got = _dense_dev(x, W, bias, act, normalize)
                want = dense_ref.dense_chain_ref(x, [(W, bias, act)], normalize)
                # gamma_n bound of an n_in-term fmaf chain and the xor tree, on sum |W x| + |b|; tanh and the
                # normalisation add a few ulps
                A = x.double().abs() @ W.double().abs().T + (0 if bias is None else bias.double().abs()[None, :])
                if normalize:
                    raw = dense_ref.dense_chain_ref(x, [(W, bias, act)], False)
                    A = A / raw.norm(dim=1, keepdim=True).clamp(min=1e-12)
                tol = (n_in + 40) * U * A + 8 * U * want.abs() + 1e-30
                err = (got.double() - want).abs()
                assert (err <= tol).all(), (act, bias is not None, normalize, float((err / tol).max()))
                again = _dense_dev(x, W, bias, act, normalize)
                assert torch.equal(got, again)
    # a row's bits do not depend on its batch: row r alone, and inside a batch at another offset
    got = _dense_dev(x, W, b, 1, True)
    for r in {0, B // 2, B - 1}:
        one = _dense_dev(x[r:r + 1].contiguous(), W, b, 1, True)
        assert torch.equal(one[0], got[r])
        pre = x[:3]
        shifted = _dense_dev(torch.cat([pre, x[r:r + 1]]).contiguous(), W, b, 1, True)
        assert torch.equal(shifted[len(pre)], got[r])


def test_dense_kernel_refuses_bad_arguments(cuda):
    from ragmeup_b200 import _lib
    x = torch.zeros((2, 8), device="cuda")
    W = torch.zeros((4, 8), device="cuda")
    y = torch.zeros((2, 4), device="cuda")
    f = _lib.lib().rmu_debug_dense
    assert f(x.data_ptr(), 2, 8, 4, W.data_ptr(), None, 2, 0, y.data_ptr(), None) == -3
    assert f(x.data_ptr(), 0, 8, 4, W.data_ptr(), None, 0, 0, y.data_ptr(), None) == -1
    assert f(x.data_ptr(), 2, 8, 0, W.data_ptr(), None, 0, 0, y.data_ptr(), None) == -1


# ------------------------------------------------------------------------------------------- encoder + Dense (golden)
@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(HERE, "golden", "distilbert.npz")))


@pytest.mark.parametrize("chain", list(G.CHAINS))
def test_tiny_distilbert_dense_matches_golden(cuda, golden, chain):
    from ragmeup_b200.encoder import BertEncoder
    cfg = G.config()
    w, chains = G.weights(cfg)
    enc = BertEncoder(cfg, {**w, **chains[chain]}, with_head=False)
    width = G.CHAINS[chain][-1][0]
    assert enc.embed_dim == width
    ids, cu = golden["ids"], golden["cu"]
    mx = int(np.diff(cu).max())
    for mode in ("mean", "cls"):
        for norm in (False, True):
            want = golden[f"{chain}_{mode}{'_norm' if norm else ''}"]
            host = enc.embed_host(ids, None, cu, mode, norm)
            dev = enc.embed_tokens(ids, None, cu, mx, mode, norm).cpu().numpy()
            assert host.shape == dev.shape == (len(cu) - 1, width)
            assert np.abs(host - want).max() < 1e-3 * max(1.0, float(np.abs(want).max())), (mode, norm)
            assert np.array_equal(host, dev)
            if norm:
                assert np.allclose(np.linalg.norm(host, axis=1), 1.0, atol=1e-5)
    # without the chain the same encoder returns the pooled rows
    plain = BertEncoder(cfg, w, with_head=False)
    got = plain.embed_host(ids, None, cu, "mean", False)
    want = golden["pooled_mean"]
    assert plain.embed_dim == cfg.hidden and np.abs(got - want).max() < 1e-3 * max(1.0, float(np.abs(want).max()))


def test_tiny_distilbert_relu_head_matches_golden(cuda, golden):
    from ragmeup_b200.encoder import BertEncoder
    cfg = G.config()
    w, _ = G.weights(cfg)
    enc = BertEncoder(cfg, w, with_head=True)
    got = enc.classify_host(golden["ids"], None, golden["cu"])
    want = golden["logits"]
    assert np.abs(got - want).max() < 2e-3 * max(1.0, float(np.abs(want).max()))


def test_set_dense_refusals(cuda):
    import ctypes as C
    from ragmeup_b200 import _lib
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import resolve_model
    cfg = DistilBertConfig(**asdict(PRESETS["tiny-distilbert"][0]))
    w = synthetic_bert_weights(cfg, seed=1)
    enc = BertEncoder(cfg, w, with_head=False)
    W = np.zeros((4, cfg.hidden), np.float32)

    def attach(h, dims, acts, Ws=None):
        dims = np.asarray(dims, np.int32)
        acts = np.asarray(acts, np.int32)
        Ws = Ws or [W] * len(acts)
        return _lib.lib().rmu_encoder_set_dense(h, len(acts), dims.ctypes.data,
                                                (C.c_void_p * len(Ws))(*[a.ctypes.data for a in Ws]),
                                                (C.c_void_p * len(Ws))(*([None] * len(Ws))), acts.ctypes.data)

    assert attach(enc._h, [cfg.hidden + 1, 4], [0]) == -1
    assert "hidden" in _lib.lib().rmu_last_error().decode()
    assert attach(enc._h, [cfg.hidden, 0], [0]) == -1
    assert attach(enc._h, [cfg.hidden, 4], [2]) == -3
    assert attach(enc._h, [cfg.hidden, 4], [1]) == 0
    assert attach(enc._h, [cfg.hidden, 4], [1]) == -1
    assert "already" in _lib.lib().rmu_last_error().decode()
    qcfg, qw, *_ = resolve_model("synthetic:tiny-qwen3", with_head=False)
    qenc = BertEncoder(qcfg, qw, with_head=False)
    assert attach(qenc._h, [qcfg.hidden, 4], [0], [np.zeros((4, qcfg.hidden), np.float32)]) == -3


# --------------------------------------------------------------------------------------------- snapshots + drop-ins
def _hf_ids(tok, texts, max_len):
    tok.enable_truncation(max_length=max_len)
    tok.no_padding()
    return [tok.encode(t.replace("\n", " ").strip()).ids for t in texts]


def _hf_pooled(model, seqs, mode):
    out = []
    with torch.no_grad():
        for s in seqs:
            h = model(input_ids=torch.tensor([s])).last_hidden_state[0]
            out.append(h[0] if mode == "cls" else h.mean(0))
    return torch.stack(out)


@pytest.fixture(scope="module")
def distil_snapshot(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("distiluse"))
    cfg = DistilBertConfig(vocab_size=1000, hidden=128, layers=2, heads=4, ffn=256, max_pos=128)
    model, layers = G.write_snapshot(path, cfg, dense=((200, True, "tanh"),), seed=3)
    return path, model, [layers[k] for k in sorted(layers)]


def _texts(n, seed):
    from ragmeup_b200.tokenizer import synthetic_sentences, synthetic_vocab
    return synthetic_sentences(synthetic_vocab(1000), n, 2, 40, seed=seed)


def test_snapshot_embeddings_store_and_similarity(cuda, distil_snapshot, monkeypatch):
    from ragmeup_b200.documents import Document
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.provenance import DocumentSimilarityAttribution
    from ragmeup_b200.vectorstore import Milvus
    path, model, layers = distil_snapshot
    emb = HuggingFaceEmbeddings(model_name=path)
    assert (emb.pooling, emb.normalize, emb.client.embed_dim, emb._types) == ("mean", False, 200, False)
    texts = _texts(40, 1) + ["line one\nline two  "]

    def encode64(ts):
        seqs = _hf_ids(emb.tokenizer, ts, emb.max_seq_length)
        return dense_ref.dense_chain_ref(_hf_pooled(model, seqs, "mean"), layers, False).numpy()

    want = encode64(texts)
    got = np.asarray(emb.embed_documents(texts), np.float32)
    assert got.shape == (len(texts), 200)
    assert np.abs(got - want).max() < 1e-3 * max(1.0, float(np.abs(want).max()))
    assert np.array_equal(np.asarray(emb.embed_query(texts[3])), got[3])
    t = emb.encode_tensor(texts).cpu().numpy()
    assert np.abs(t - got).max() < 1e-6
    assert emb.encode_tensor([]).shape == (0, 200) and np.asarray(emb._encode_host([])).shape == (0, 200)
    # a vector store over the projected vectors finds each document by its own text
    store = Milvus(emb)
    store.add_documents([Document(page_content=x) for x in texts[:20]])
    for i in (0, 7, 19):
        assert store.similarity_search(texts[i], k=1)[0].page_content == texts[i]
    # DocumentSimilarityAttribution against the reference's compute_similarity restated in float64
    docs = [Document(page_content=x) for x in texts[:6]]
    query, answer = texts[30], texts[31]
    attr = DocumentSimilarityAttribution(embeddings=emb)
    for setting, include in (("True", True), ("False", False)):
        monkeypatch.setenv("attribute_include_query", setting)
        got_s = np.asarray(attr.compute_similarity(query, docs, answer), np.float64)
        want_s = np.asarray(provenance_ref.compute_similarity(encode64, query, texts[:6], answer, include), np.float64)
        assert np.abs(got_s - want_s).max() < 1e-3 * max(1.0, float(np.abs(want_s).max())), setting


def test_snapshot_cross_encoder_relu_head_no_token_types(cuda, tmp_path):
    """pairs send no token types (type id 1 would index past DistilBERT's one-row table) and score as transformers'
    DistilBertForSequenceClassification does, through a sigmoid for its one label"""
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    cfg = DistilBertConfig(vocab_size=1000, hidden=128, layers=2, heads=4, ffn=256, max_pos=128, num_labels=1)
    model, _ = G.write_snapshot(str(tmp_path), cfg, head=True, seed=4)
    ce = HuggingFaceCrossEncoder(model_name=str(tmp_path))
    assert ce._types is False and ce.activation == "sigmoid"
    texts = _texts(24, 2)
    pairs = [(texts[i], texts[i + 12]) for i in range(12)]
    got = ce.score(pairs)
    tok = ce.tokenizer
    tok.enable_truncation(max_length=ce.max_length, strategy="longest_first")
    tok.no_padding()
    with torch.no_grad():
        logits = torch.cat([model(input_ids=torch.tensor([tok.encode(a, b).ids])).logits[:, 0] for a, b in pairs])
    want = torch.sigmoid(logits).numpy()
    assert np.abs(got - want).max() < 1e-3
    assert np.abs(ce.score_tensor(pairs).cpu().numpy() - got).max() < 1e-6


def test_labse_shape_cls_dense_normalize_matches_oracle(cuda):
    """a LaBSE-shaped BERT (768 / 12 heads / 3072, two layers, small vocabulary): CLS pooling, Dense 768 -> 768 tanh,
    Normalize, against the float64 encoder oracle and the float64 Dense chain"""
    from ragmeup_b200.encoder import BertEncoder
    cfg = BertConfig(**{**asdict(PRESETS["LaBSE"][0]), "vocab_size": 2000, "layers": 2})
    w = synthetic_bert_weights(cfg, seed=8)
    dw = synthetic_dense_weights(cfg.hidden, ((768, True, "tanh"),), seed=8)
    enc = BertEncoder(cfg, {**w, **dw}, with_head=False)
    rng = np.random.default_rng(2)
    lens = [1, 5, 64, 256, 17]
    ids = np.concatenate([np.r_[101, rng.integers(200, 2000, n - 1)] for n in lens]).astype(np.int32)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    got = enc.embed_host(ids, np.zeros_like(ids), cu, "cls", True)
    wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    cls = ref.encoder_stack_ref(wd, cfg, ids, None, cu, "split", device="cuda")["cls"]
    want = dense_ref.dense_chain_ref(cls, dense_layers(dw), True).cpu().numpy()
    assert got.shape == (len(lens), 768)
    assert np.abs(got - want).max() < 1e-3 * max(1.0, float(np.abs(want).max()))
