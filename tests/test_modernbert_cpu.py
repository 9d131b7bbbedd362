"""ModernBERT on the host, no GPU: config parsing in both config.json forms and the refusals by field name, the rope
tables against transformers, the fp32 oracle against transformers' ModernBERT, the canonical weights, tokenisation, and
the C ABI's refusals before any CUDA call."""
from __future__ import annotations

import ctypes as C
import json
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import modernbert_ref as mr
from ragmeup_b200.weights import (PRESETS, ModernBertConfig, load_hf_snapshot, modernbert_to_canonical,
                                  modernbert_weight_names, resolve_flashrank, resolve_model, rope_tables,
                                  synthetic_bert_weights)

RELEASE = {"model_type": "modernbert", "vocab_size": 1000, "hidden_size": 128, "num_hidden_layers": 7,
           "num_attention_heads": 2, "intermediate_size": 192, "max_position_embeddings": 1024, "norm_eps": 1e-5,
           "global_attn_every_n_layers": 3, "global_rope_theta": 160000.0, "local_rope_theta": 10000.0,
           "local_attention": 128, "classifier_pooling": "mean", "hidden_activation": "gelu",
           "classifier_activation": "gelu"}


def test_release_config_form():
    cfg = ModernBertConfig.from_hf(RELEASE)
    assert cfg.layer_windows == (0, 64, 64, 0, 64, 64, 0)
    assert (cfg.global_theta, cfg.local_theta, cfg.classifier_pooling) == (160000.0, 10000.0, "mean")
    assert (cfg.hidden, cfg.layers, cfg.heads, cfg.ffn, cfg.max_pos) == (128, 7, 2, 192, 1024)


def test_transformers5_config_form():
    d = {k: v for k, v in RELEASE.items() if k not in ("global_attn_every_n_layers", "global_rope_theta",
                                                       "local_rope_theta")}
    d["layer_types"] = ["full_attention", "sliding_attention", "full_attention", "sliding_attention",
                        "sliding_attention", "sliding_attention", "full_attention"]
    d["rope_parameters"] = {"full_attention": {"rope_type": "default", "rope_theta": 80000.0},
                            "sliding_attention": {"rope_type": "default", "rope_theta": 5000.0}}
    d["local_attention"] = 32
    cfg = ModernBertConfig.from_hf(d)
    assert cfg.layer_windows == (0, 16, 0, 16, 16, 16, 0)
    assert (cfg.global_theta, cfg.local_theta) == (80000.0, 5000.0)


def test_transformers_config_round_trip():
    transformers = pytest.importorskip("transformers")
    hc = transformers.ModernBertConfig(vocab_size=1000, hidden_size=128, num_hidden_layers=5, num_attention_heads=2,
                                       intermediate_size=192, local_attention=64, global_attn_every_n_layers=2,
                                       pad_token_id=0, bos_token_id=1, eos_token_id=2, cls_token_id=1, sep_token_id=2)
    cfg = ModernBertConfig.from_hf(hc.to_dict())
    assert cfg.layer_windows == tuple(0 if t == "full_attention" else 32 for t in hc.layer_types)
    assert cfg.global_theta == 160000.0 and cfg.local_theta == 10000.0


@pytest.mark.parametrize("field,value", [("hidden_activation", "gelu_pytorch_tanh"), ("classifier_activation", "silu"),
                                         ("classifier_pooling", "max"),
                                         ("rope_parameters", {"full_attention": {"rope_type": "yarn", "factor": 2.0}}),
                                         ("rope_scaling", {"rope_type": "linear", "factor": 2.0}),
                                         ("layer_types", ["full_attention", "chunked_attention"] * 3 + ["full_attention"]),
                                         ("head_dim", 32)])
def test_refusals_name_the_field(field, value):
    name = "rope_type" if field == "rope_parameters" else field
    with pytest.raises(ValueError, match=name):
        ModernBertConfig.from_hf({**RELEASE, field: value})


def test_rope_tables_equal_transformers():
    transformers = pytest.importorskip("transformers")
    from transformers.models.modernbert.modeling_modernbert import ModernBertRotaryEmbedding
    cfg = ModernBertConfig(hidden=768, heads=12, layers=3, ffn=1152, max_pos=8192)
    hc = transformers.ModernBertConfig(hidden_size=768, num_attention_heads=12, num_hidden_layers=3,
                                       intermediate_size=1152, max_position_embeddings=8192)
    rot = ModernBertRotaryEmbedding(hc)
    pos = torch.arange(8192)[None]
    x = torch.zeros(1, dtype=torch.float32)
    tabs = rope_tables(cfg)
    for i, t in enumerate(("full_attention", "sliding_attention")):
        cos, sin = rot(x, pos, layer_type=t)
        assert np.array_equal(cos[0, :, :32].numpy(), tabs[2 * i]) and np.array_equal(cos[0, :, 32:].numpy(), tabs[2 * i])
        assert np.array_equal(sin[0, :, :32].numpy(), tabs[2 * i + 1])


def _hf_model(cfg, w, pooling):
    transformers = pytest.importorskip("transformers")
    windows = set(x for x in cfg.layer_windows if x)
    hc = transformers.ModernBertConfig(
        vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, num_hidden_layers=cfg.layers,
        num_attention_heads=cfg.heads, intermediate_size=cfg.ffn, max_position_embeddings=cfg.max_pos,
        layer_types=["full_attention" if x == 0 else "sliding_attention" for x in cfg.layer_windows],
        local_attention=2 * (windows.pop() if windows else 64), classifier_pooling=pooling, pad_token_id=0,
        bos_token_id=1, eos_token_id=2, cls_token_id=1, sep_token_id=2, num_labels=cfg.num_labels,
        attn_implementation="eager")
    m = transformers.ModernBertForSequenceClassification(hc).eval()
    sd = {}
    for k, v in w.items():
        if k.startswith("layers.0.attn_norm") or (k.endswith(".bias") and not k.startswith("classifier")):
            continue                                   # no such tensors in the model (all biases false)
        sd[k if k.startswith(("head.", "classifier.")) else "model." + k] = torch.from_numpy(v)
    m.load_state_dict(sd, strict=True)
    return m


@pytest.mark.parametrize("preset,pooling", [("tiny-modernbert", "cls"), ("tiny-modernbert-window", "mean")])
def test_oracle_matches_transformers(preset, pooling):
    """the fp32 oracle against transformers' ModernBertForSequenceClassification (eager attention), lengths across the
    window and past 600 tokens"""
    cfg = ModernBertConfig(**asdict(PRESETS[preset][0]))
    cfg.classifier_pooling = pooling
    w = synthetic_bert_weights(cfg, seed=4, with_head=True, scale=4.0)
    m = _hf_model(cfg, w, pooling)
    rng = np.random.default_rng(0)
    lens = [17, 65, 66, 129, 640]
    ids = np.concatenate([rng.integers(3, cfg.vocab_size, n) for n in lens])
    cu = np.r_[0, np.cumsum(lens)]
    got = mr.modernbert_stack(w, cfg, ids, cu, torch.float32)
    with torch.no_grad():
        for b, n in enumerate(lens):
            out = m(torch.from_numpy(ids[cu[b]:cu[b + 1]])[None], output_hidden_states=True)
            h = out.hidden_states[-1][0]
            assert float((got["hidden"][cu[b]:cu[b + 1]] - h).abs().max()) < 2e-4 * max(1.0, float(h.abs().max()))
            assert abs(float(got["logits"][b, 0]) - float(out.logits[0, 0])) < 1e-4 * max(1.0, abs(float(out.logits[0, 0])))
    f64 = mr.modernbert_stack(w, cfg, ids, cu, torch.float64)
    assert float((f64["logits"] - got["logits"].double()).abs().max()) < 1e-3


def _golden_script():
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden_modernbert.py")
    spec = importlib.util.spec_from_file_location("make_golden_modernbert", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _golden_case(g, gm, case):
    preset, seed, scale, pooling, lens = case
    key = gm.case_key(preset, seed, scale, pooling)
    cfg = gm.case_config(preset, pooling)
    w = synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale)
    mask = g[key + "_mask"]
    assert mask.sum(1).tolist() == lens
    ids = np.concatenate([g[key + "_ids"][b, :n] for b, n in enumerate(lens)])
    return key, cfg, w, ids, np.r_[0, np.cumsum(lens)]


@pytest.mark.parametrize("case", range(4))
def test_oracle_matches_goldens(golden_dir, case):
    """the fp32 and float64 oracles against transformers' ModernBertForSequenceClassification outputs stored in
    tests/golden/modernbert.npz: both tiny presets, CLS and mean pooling, lengths 65 / 66 / 129 / 161 and past 600"""
    gm = _golden_script()
    g = np.load(f"{golden_dir}/modernbert.npz")
    key, cfg, w, ids, cu = _golden_case(g, gm, gm.CASES[case])
    last = cu[1:] - 1
    for dtype, tol in ((torch.float32, 2e-5), (torch.float64, 1e-4)):
        got = mr.modernbert_stack(w, cfg, ids, cu, dtype)
        h = got["hidden"].double()
        want_logits = g[key + "_logits"]
        scale = max(1.0, float(np.abs(want_logits).max()))
        assert np.abs(got["logits"].double().numpy() - want_logits).max() < tol * scale, dtype
        assert np.abs(h[cu[:-1]].numpy() - g[key + "_h_first"]).max() < tol * 10, dtype
        assert np.abs(h[last].numpy() - g[key + "_h_last"]).max() < tol * 10, dtype
        mean = np.stack([h[cu[b]:cu[b + 1]].mean(0).numpy() for b in range(len(cu) - 1)])
        assert np.abs(mean - g[key + "_h_mean"]).max() < tol * 10, dtype


def test_golden_script_reproduces_the_fixture(golden_dir):
    """rerunning tests/golden/make_golden_modernbert.py gives the stored arrays"""
    pytest.importorskip("transformers")
    gm = _golden_script()
    g = np.load(f"{golden_dir}/modernbert.npz")
    fresh = gm.modernbert_goldens()
    assert sorted(fresh) == sorted(g.files)
    for k, v in fresh.items():
        if k.endswith(("_ids", "_mask")):
            assert np.array_equal(v, g[k]), k
        else:
            np.testing.assert_allclose(v, g[k], rtol=0, atol=1e-5, err_msg=k)


def test_canonical_weights_fill_absent_tensors():
    cfg = ModernBertConfig(**asdict(PRESETS["tiny-modernbert"][0]))
    w = synthetic_bert_weights(cfg, seed=0, with_head=True)
    raw = {("model." + k if not k.startswith(("head.", "classifier.")) else k): v for k, v in w.items()
           if not k.endswith(".bias") or k.startswith("classifier.")}
    raw = {k: v for k, v in raw.items() if not k.startswith("model.layers.0.attn_norm")}
    raw["decoder.bias"] = np.zeros(cfg.vocab_size, np.float32)
    c = modernbert_to_canonical(raw, cfg, True)
    assert "decoder.bias" not in c
    for name, shape in modernbert_weight_names(cfg, True):
        assert c[name].shape == shape, name
        np.testing.assert_array_equal(c[name], w[name])


def test_presets_resolve():
    cfg, w, pooling, normalize, max_len, act, src = resolve_model("synthetic:modernbert-embed-base", with_head=False)
    assert isinstance(cfg, ModernBertConfig) and pooling == "mean" and normalize and max_len == 8192
    assert cfg.layer_windows.count(0) == 8 and len(cfg.layer_windows) == 22
    cfg, *_, act, _src = resolve_model("synthetic:gte-reranker-modernbert-base", with_head=True)
    assert act == "sigmoid" and cfg.num_labels == 1
    assert not resolve_model("synthetic:gte-modernbert-base", with_head=False)[3]
    large = PRESETS["modernbert-large"][0]
    assert (large.hidden, large.layers, large.heads, large.ffn) == (1024, 28, 16, 2624)
    with pytest.raises(ValueError, match="FlashRank"):
        resolve_flashrank("synthetic:tiny-modernbert")


def test_tokenisation(tmp_path):
    from ragmeup_b200.tokenizer import PairAssembler, load_tokenizer
    tok = load_tokenizer(None, 1000, modernbert=True)
    ids, _typ, cu = PairAssembler(tok, 64)(["ba ce"], ["di fo gu"])
    v = tok.get_vocab()
    assert ids[0] == v["[CLS]"] and ids[cu[1] - 1] == v["[SEP]"] and list(ids).count(v["[SEP]"]) == 2
    tok.save(str(tmp_path / "tokenizer.json"))
    assert load_tokenizer(str(tmp_path), 1000, modernbert=True).to_str() == tok.to_str()
    with pytest.raises(FileNotFoundError, match="tokenizer.json"):
        load_tokenizer(str(tmp_path / "nowhere"), 1000, modernbert=True)


def test_snapshot_config_is_authoritative(tmp_path):
    from safetensors.numpy import save_file
    cfg = ModernBertConfig.from_hf(RELEASE)
    w = synthetic_bert_weights(cfg, seed=0, with_head=False)
    save_file({"model." + k: v for k, v in w.items() if not k.endswith(".bias") and "layers.0.attn_norm" not in k},
              str(tmp_path / "model.safetensors"))
    (tmp_path / "config.json").write_text(json.dumps(RELEASE))
    got, wl, pooling, normalize, max_len, act = load_hf_snapshot(str(tmp_path), with_head=False)
    assert got.layer_windows == cfg.layer_windows and max_len == 1024 and pooling == "mean"
    assert set(wl) >= {n for n, _ in modernbert_weight_names(cfg, False)}


def _create(cfg, windows, pooling=1, head_form=0, rope_rows=None, rope_half=None, n=None, nulls=()):
    from ragmeup_b200 import _lib
    win = np.ascontiguousarray(windows, dtype=np.int32)
    mb = _lib.ModernBertExtC(win.ctypes.data, pooling, head_form, cfg.max_pos if rope_rows is None else rope_rows,
                             cfg.head_dim // 2 if rope_half is None else rope_half)
    count = 3 + 12 * cfg.layers + 2 + 4 if n is None else n
    dummy = np.zeros(1, np.float32)
    ptrs = (C.c_void_p * count)(*[None if i in nulls else dummy.ctypes.data for i in range(count)])
    h = C.c_void_p()
    cc = _lib.bert_config_c(cfg)
    return _lib.lib().rmu_encoder_create_modernbert(C.byref(cc), C.byref(mb), ptrs, count, 0, C.byref(h))


def test_c_refusals_before_any_cuda_call():
    """every refusal returns before the weights are read or a CUDA call is made (the tensors here are 1-element
    dummies, and the machine may have no GPU)"""
    from dataclasses import replace
    ERR_ARG, UNSUP = -1, -3
    cfg = ModernBertConfig(**asdict(PRESETS["tiny-modernbert"][0]))
    win = list(cfg.layer_windows)
    assert _create(replace(cfg, hidden=128, heads=1), win) == UNSUP                # d_h = 128
    assert _create(replace(cfg, ffn=160), win) == UNSUP                           # F % 64
    assert _create(cfg, win, head_form=1) == UNSUP
    assert _create(cfg, [0, -1, 64, 0]) == ERR_ARG                                # negative window
    assert _create(cfg, win, pooling=7) == ERR_ARG
    assert _create(cfg, win, rope_rows=cfg.max_pos - 1) == ERR_ARG                # wrong table size
    assert _create(cfg, win, rope_half=cfg.head_dim) == ERR_ARG
    assert _create(cfg, win, n=3 + 12 * cfg.layers + 2 + 3) == ERR_ARG          # a rope table missing
    n = 3 + 12 * cfg.layers + 2 + 4
    assert _create(cfg, win, nulls=(n - 1,)) == ERR_ARG                           # null rope table
    assert _create(cfg, win, nulls=(5,)) == ERR_ARG                               # null Wqkv

    class WithAdapter(ModernBertConfig):
        adapter_dim = 128

    class WithRel(ModernBertConfig):
        rel_buckets = 32
    assert _create(WithAdapter(**asdict(cfg)), win) == UNSUP
    assert _create(WithRel(**asdict(cfg)), win) == UNSUP


def test_c_refuses_gemm_weights_the_split_planes_cannot_hold():
    """GEMM weights travel as split fp16 planes: |w| >= 65520 is refused on the host, before any CUDA call, with its
    index in the checkpoint's layout (Wi's is taken before the GeGLU row blocks reorder it)"""
    from ragmeup_b200 import _lib
    cfg = ModernBertConfig(**asdict(PRESETS["tiny-modernbert"][0]))
    names = [n for n, _ in modernbert_weight_names(cfg, False)]
    arrs = [np.zeros(shape, np.float32) for _, shape in modernbert_weight_names(cfg, False)]
    arrs += [np.ascontiguousarray(t, dtype=np.float32) for t in rope_tables(cfg)]
    ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    win = np.ascontiguousarray(cfg.layer_windows, dtype=np.int32)
    mb = _lib.ModernBertExtC(win.ctypes.data, 1, 0, cfg.max_pos, cfg.head_dim // 2)

    def create():
        h = C.c_void_p()
        rc = _lib.lib().rmu_encoder_create_modernbert(C.byref(_lib.bert_config_c(cfg)), C.byref(mb), ptrs, len(arrs), 0,
                                                      C.byref(h))
        if rc == 0:
            _lib.lib().rmu_encoder_destroy(h)
        return rc

    wi = arrs[names.index("layers.1.mlp.Wi.weight")].reshape(-1)
    j = cfg.ffn * cfg.hidden + 5                                       # a gate row, which the GeGLU blocks move
    for v in (7e4, -65520.0, np.inf):
        wi[j] = v
        assert create() == -3, v
        msg = _lib.lib().rmu_last_error().decode()
        assert "65520" in msg and f"layer 1 mlp Wi weight [{j}]" in msg, msg
    wi[j] = 65519.0
    assert create() in (0, -2)                                         # accepted: without a device the next step fails
