"""DistilBERT snapshots and sentence-transformers Dense modules without a device: the config mapping and tensor
renaming against snapshots saved by transformers, the float64 oracle against transformers' DistilBERT, modules.json
parsing and its refusals, the golden fixture's regeneration, DocumentSimilarityAttribution's host arithmetic, and the
C entry points' refusals."""
import ctypes
import importlib.util
import json
import os
import shutil
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import dense_ref
from oracle import encoder_kernels_ref as ref
from ragmeup_b200.weights import (MODEL_TYPES, PRESETS, DistilBertConfig, dense_layers, load_hf_snapshot,
                                  resolve_colbert, resolve_flashrank, resolve_model, weight_names)

HERE = os.path.dirname(os.path.abspath(__file__))
CFG = DistilBertConfig(vocab_size=1000, hidden=128, layers=2, heads=4, ffn=256, max_pos=128)


def _golden_module(name="make_golden_distilbert"):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, "golden", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def G():
    pytest.importorskip("transformers")
    return _golden_module()


def _snap(G, tmp_path, name="s", **kw):
    path = str(tmp_path / name)
    os.makedirs(path, exist_ok=True)
    model, layers = G.write_snapshot(path, CFG if not kw.get("head") else DistilBertConfig(**{**asdict(CFG),
                                                                                              "num_labels": 1}), **kw)
    return path, model, layers


# ------------------------------------------------------------------------------------------------------- config
def test_config_mapping_and_refusal():
    d = {"model_type": "distilbert", "vocab_size": 119547, "dim": 768, "n_layers": 6, "n_heads": 12,
         "hidden_dim": 3072, "max_position_embeddings": 512, "activation": "gelu", "sinusoidal_pos_embds": False}
    c = DistilBertConfig.from_hf(d)
    assert asdict(c) == asdict(PRESETS["distiluse-base-multilingual-cased-v2"][0])
    assert (c.ln_eps, c.type_vocab, c.head_act, c.position_mode, c.num_labels) == (1e-12, 1, 2, 0, 1)
    assert DistilBertConfig.from_hf({**d, "id2label": {0: "a", 1: "b"}}).num_labels == 2
    with pytest.raises(ValueError, match="activation"):
        DistilBertConfig.from_hf({**d, "activation": "relu"})
    with pytest.raises(ValueError, match="distilbert config.json without 'dim'"):
        DistilBertConfig.from_hf({k: v for k, v in d.items() if k != "dim"})
    assert "distilbert" in MODEL_TYPES


@pytest.mark.parametrize("sinusoidal", [False, True])
def test_snapshot_renaming_and_oracle_equal_transformers(G, tmp_path, sinusoidal):
    path, model, layers = _snap(G, tmp_path, dense=((200, True, "tanh"), (50, False, "identity")), normalize=True,
                                sinusoidal=sinusoidal)
    cfg, w, pooling, normalize, max_len, act = load_hf_snapshot(path, with_head=False)
    assert type(cfg) is DistilBertConfig and asdict(cfg) == asdict(CFG)
    assert (pooling, normalize, max_len, act) == ("mean", True, 128, "identity")
    sd = {k: v.numpy() for k, v in model.float().state_dict().items()}
    model.double()
    for name, shape in weight_names(cfg, False):
        assert w[name].shape == shape, name
    assert not w["embeddings.token_type_embeddings.weight"].any()
    assert np.array_equal(w["embeddings.position_embeddings.weight"], sd["embeddings.position_embeddings.weight"])
    assert np.array_equal(w["encoder.layer.1.attention.self.key.weight"], sd["transformer.layer.1.attention.k_lin.weight"])
    assert np.array_equal(w["encoder.layer.0.attention.output.LayerNorm.bias"], sd["transformer.layer.0.sa_layer_norm.bias"])
    assert np.array_equal(w["encoder.layer.0.output.dense.weight"], sd["transformer.layer.0.ffn.lin2.weight"])
    assert np.array_equal(w["encoder.layer.1.output.LayerNorm.weight"], sd["transformer.layer.1.output_layer_norm.weight"])
    # the float64 BERT oracle on the renamed weights, and the Dense chain, equal transformers' DistilBertModel
    got_layers = dense_layers(w)
    assert [(a.shape, b is None, c) for a, b, c in got_layers] == [((200, 128), False, 1), ((50, 200), True, 0)]
    lens = [1, 7, 30]
    rng = np.random.default_rng(0)
    ids = np.concatenate([np.r_[101, rng.integers(5, 1000, n - 1)] for n in lens]).astype(np.int32)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    out = ref.encoder_stack_ref(w, cfg, ids, None, cu)
    with torch.no_grad():
        hs = [model(input_ids=torch.tensor(ids[cu[b]:cu[b + 1]][None]).long()).last_hidden_state[0]
              for b in range(len(lens))]
    assert float((torch.cat(hs) - out["hidden"]).abs().max()) < 1e-12
    mine = dense_ref.dense_chain_ref(out["mean"], got_layers, True)
    want = torch.stack([h.mean(0) for h in hs])
    for Wd, bd, a in [layers[k] for k in sorted(layers)]:
        want = want @ torch.from_numpy(Wd).double().T + (0 if bd is None else torch.from_numpy(bd).double())
        want = torch.tanh(want) if a == 1 else want
    want = want / want.norm(dim=1, keepdim=True)
    assert float((mine - want).abs().max()) < 1e-12


def test_head_snapshot_relu_head_equals_transformers(G, tmp_path):
    path, model, _ = _snap(G, tmp_path, head=True)
    cfg, w, _p, _n, _l, act = load_hf_snapshot(path, with_head=True)
    assert act == "sigmoid" and cfg.num_labels == 1 and cfg.head_act == 2
    sd = {k: v.numpy() for k, v in model.float().state_dict().items()}
    model.double()
    assert np.array_equal(w["pooler.dense.weight"], sd["pre_classifier.weight"])
    assert np.array_equal(w["classifier.bias"], sd["classifier.bias"])
    ids = np.array([101, 9, 44, 102, 77, 102, 101, 5, 102], np.int32)
    cu = np.array([0, 6, 9], np.int32)
    h = ref.encoder_stack_ref(w, cfg, ids, None, cu)["hidden"]
    mine = dense_ref.relu_head_ref(h[[0, 6]], w["pooler.dense.weight"], w["pooler.dense.bias"], w["classifier.weight"],
                                   w["classifier.bias"])
    with torch.no_grad():
        want = torch.cat([model(input_ids=torch.tensor(ids[a:b][None]).long()).logits for a, b in ((0, 6), (6, 9))])
    assert float((mine - want).abs().max()) < 1e-12
    with open(os.path.join(path, "config.json")) as f:
        d = json.load(f)
    d["sbert_ce_default_activation_function"] = "torch.nn.modules.linear.Identity"
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(d, f)
    assert load_hf_snapshot(path, with_head=True)[5] == "identity"


def test_dense_weight_file_forms_agree(G, tmp_path):
    a, _, la = _snap(G, tmp_path, "a", dense=((64, True, "tanh"),), dense_format="safetensors", seed=2)
    b, _, lb = _snap(G, tmp_path, "b", dense=((64, True, "tanh"),), dense_format="bin", seed=2)
    wa, wb = load_hf_snapshot(a, False)[1], load_hf_snapshot(b, False)[1]
    for (Wa, ba, xa), (Wb, bb, xb) in zip(dense_layers(wa), dense_layers(wb)):
        assert np.array_equal(Wa, Wb) and np.array_equal(ba, bb) and xa == xb == 1
    assert np.array_equal(dense_layers(wa)[0][0], la["2_Dense"][0])


def _edit_modules(path, fn):
    p = os.path.join(path, "modules.json")
    with open(p) as f:
        mods = json.load(f)
    with open(p, "w") as f:
        json.dump(fn(mods), f)


def _edit_dense_config(path, mdir, **kw):
    p = os.path.join(path, mdir, "config.json")
    with open(p) as f:
        d = json.load(f)
    with open(p, "w") as f:
        json.dump({**d, **kw}, f)


@pytest.mark.parametrize("kind", ["LayerNorm", "CNN", "LSTM", "WeightedLayerPooling"])
def test_unknown_module_types_are_refused(G, tmp_path, kind):
    path, _, _ = _snap(G, tmp_path)
    _edit_modules(path, lambda m: m + [{"idx": 9, "name": "9", "path": f"9_{kind}",
                                        "type": f"sentence_transformers.models.{kind}"}])
    with pytest.raises(ValueError, match=f"9_{kind}.*{kind}"):
        load_hf_snapshot(path, with_head=False)
    # a BERT snapshot is read the same way: no module is skipped without a word
    with open(os.path.join(path, "config.json")) as f:
        d = json.load(f)
    with pytest.raises(ValueError, match=kind):
        resolve_model(path, with_head=False)
    assert d["model_type"] == "distilbert"


def test_dense_refusals_name_their_field(G, tmp_path):
    path, _, _ = _snap(G, tmp_path, dense=((64, True, "tanh"), (32, True, "tanh")), normalize=True)
    base = str(tmp_path / "base")
    shutil.copytree(path, base)

    def fresh():
        shutil.rmtree(path)
        shutil.copytree(base, path)

    _edit_dense_config(path, "3_Dense", activation_function="torch.nn.modules.activation.ReLU")
    with pytest.raises(ValueError, match="3_Dense.*activation_function"):
        load_hf_snapshot(path, with_head=False)
    fresh()
    _edit_dense_config(path, "3_Dense", in_features=65)
    with pytest.raises(ValueError, match="3_Dense.*in_features"):
        load_hf_snapshot(path, with_head=False)
    fresh()
    _edit_modules(path, lambda m: [m[0], m[2], m[1], m[3], m[4]])          # Dense before Pooling
    with pytest.raises(ValueError, match="2_Dense.*before Pooling"):
        load_hf_snapshot(path, with_head=False)
    fresh()
    _edit_modules(path, lambda m: [m[0], m[1], m[2], m[4], m[3]])          # Normalize before a Dense
    with pytest.raises(ValueError, match="Normalize comes before Dense module '3_Dense'"):
        load_hf_snapshot(path, with_head=False)
    fresh()
    _edit_dense_config(path, "2_Dense", bias=False)
    with pytest.raises(ValueError, match="2_Dense.*bias"):
        load_hf_snapshot(path, with_head=False)
    fresh()
    assert [W.shape for W, _b, _a in dense_layers(load_hf_snapshot(path, with_head=False)[1])] == [(64, 128), (32, 64)]


def test_dense_in_a_qwen3_snapshot_is_refused(tmp_path):
    pytest.importorskip("transformers")
    mod = _golden_module("make_golden_qwen3")
    cfg, w, lm, tok = mod.build()
    snaps = mod.save_snapshots(str(tmp_path / "q"), cfg, w, lm, tok)
    path = snaps["embedder"]
    _edit_modules(path, lambda m: [x for x in m if not x["type"].endswith("Normalize")] +
                  [{"path": "2_Dense", "type": "sentence_transformers.models.Dense"}])
    with pytest.raises(ValueError, match="Dense module '2_Dense' in a Qwen3 snapshot"):
        load_hf_snapshot(path, with_head=False)


def test_colbert_and_flashrank_refuse_distilbert(G, tmp_path):
    path, _, _ = _snap(G, tmp_path, head=True)
    assert resolve_colbert(path) is None                                  # a cross-encoder, not ColBERT
    with open(os.path.join(path, "config.json")) as f:
        d = json.load(f)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump({**d, "architectures": ["HF_ColBERT"]}, f)
    with pytest.raises(ValueError, match="ColBERT checkpoint of model_type 'distilbert'"):
        resolve_colbert(path)
    with pytest.raises(ValueError, match="DistilBERT.*not a FlashRank model"):
        resolve_flashrank("synthetic:tiny-distilbert")


def test_presets():
    cfg, w, pooling, normalize, max_len, act, src = resolve_model("synthetic:tiny-distilbert", with_head=False)
    assert (type(cfg), pooling, normalize, max_len, src) == (DistilBertConfig, "mean", False, 64, None)
    assert [(W.shape, b.shape, a) for W, b, a in dense_layers(w)] == [((200, 128), (200,), 1)]
    assert resolve_model("synthetic:tiny-distilbert", with_head=True)[5] == "sigmoid"
    for name, (cfg, pooling, n) in (("distiluse-base-multilingual-cased-v2", (DistilBertConfig, "mean", 128)),
                                    ("LaBSE", (type(PRESETS["LaBSE"][0]), "cls", 256))):
        c, p, m = PRESETS[name]
        assert (type(c), p, m) == (cfg, pooling, n)
    assert PRESETS["LaBSE"][0].vocab_size == 501153 and PRESETS["distiluse-base-multilingual-cased-v2"][0].vocab_size == 119547


# ------------------------------------------------------------------------------------------------------- fixture
def test_fixture_regenerates_bit_for_bit(G):
    want = np.load(os.path.join(HERE, "golden", "distilbert.npz"))
    got = G.make()
    assert sorted(got) == sorted(want.files)
    for k in want.files:
        assert np.array_equal(got[k], want[k]), k


# ------------------------------------------------------------------------------------ similarity host arithmetic
@pytest.mark.parametrize("setting", ["True", "False"])
def test_similarity_attribution_host_arithmetic(monkeypatch, setting):
    """compute_similarity's arithmetic after the encoder and the cosine search, with a stand-in encoder and index,
    against the reference's compute_similarity restated in float64 with sklearn's cosine_similarity"""
    from sklearn.metrics.pairwise import cosine_similarity
    from ragmeup_b200 import provenance

    rng = np.random.default_rng(3)
    table = {f"t{i}": rng.standard_normal(512).astype(np.float32) for i in range(8)}

    class Emb:
        def encode_tensor(self, texts):
            return torch.from_numpy(np.stack([table[t] for t in texts]))

    class Index:
        def __init__(self, dim, metric, device=None):
            assert metric == "cosine"
            self.x = None

        def add(self, x):
            self.x = x.double().numpy()

        def search(self, q, k):
            s = cosine_similarity(q.double().numpy(), self.x)
            order = np.argsort(-s, axis=1, kind="stable")[:, :k]
            return torch.from_numpy(np.take_along_axis(s, order, 1)), torch.from_numpy(order)

    monkeypatch.setattr(provenance, "FlatIndex", Index)
    monkeypatch.setenv("attribute_include_query", setting)
    docs = [f"t{i}" for i in range(6)]
    got = provenance.DocumentSimilarityAttribution(embeddings=Emb()).compute_similarity("t6", docs, "t7")
    enc = lambda ts: np.stack([table[t] for t in ts]).astype(np.float64)  # noqa: E731
    a, q = enc(["t7"]), enc(["t6"])
    sims = []
    for d in enc(docs):
        s = cosine_similarity([d], a)[0][0]
        sims.append((s + cosine_similarity([d], q)[0][0]) / 2 if setting == "True" else s)
    total = sum(sims)
    want = [s / total for s in sims] if total > 0 else sims
    assert np.abs(np.asarray(got, np.float64) - np.asarray(want)).max() < 1e-6


# ---------------------------------------------------------------------------------------------------- C refusals
def test_c_entry_points_refuse_bad_arguments():
    from ragmeup_b200 import _lib
    L = _lib.lib()
    dims = np.array([128, 4], np.int32)
    acts = np.array([0], np.int32)
    W = np.zeros((4, 128), np.float32)
    ws = (ctypes.c_void_p * 1)(W.ctypes.data)
    assert L.rmu_encoder_set_dense(None, 1, dims.ctypes.data, ws, None, acts.ctypes.data) == -1
    assert "set_dense" in L.rmu_last_error().decode()
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data
    assert L.rmu_debug_dense(None, 2, 8, 4, p, None, 0, 0, p, None) == -1
    assert L.rmu_debug_dense(p, 2, 0, 4, p, None, 0, 0, p, None) == -1
    assert L.rmu_debug_dense(p, 2, 8, 4, p, None, 2, 0, p, None) == -3
    assert "RMU_DENSE_TANH" in L.rmu_last_error().decode()
    # RMU_HEAD_RELU is DistilBERT's head: another value, or ReLU with disentangled attention, is refused before any
    # CUDA call
    from ragmeup_b200.weights import synthetic_bert_weights
    w = synthetic_bert_weights(CFG, seed=0, with_head=True)
    arrs = [w[n] for n, _ in weight_names(CFG, True)]
    ptrs = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    cc = _lib.bert_config_c(CFG)
    h = ctypes.c_void_p()
    for ext in (_lib.EncoderExtC(0, 0, 3), _lib.EncoderExtC(256, 512, 2)):
        assert L.rmu_encoder_create_ex(ctypes.byref(cc), ctypes.byref(ext), ptrs, len(arrs), 1, ctypes.byref(h)) == -3
    assert "RMU_HEAD_RELU" in L.rmu_last_error().decode()
    hi = np.zeros(64, np.uint16)
    cu = np.array([0, 1], np.int32)
    assert L.rmu_debug_cls_head_act(hi.ctypes.data, hi.ctypes.data, cu.ctypes.data, 1, 8, 1, p, p, p, p, 3, p,
                                    None) == -1
