"""CPU: MPNet sentence embedders (all-mpnet-base-v2, HuggingFaceEmbeddings' default model).  The oracles against the
goldens minted from transformers' MPNetModel (tests/golden/make_golden_mpnet.py), the host-built attention bias table
against transformers' bucket function, snapshot resolution and its refusals, the synthetic MPNet tokenizer, and the
C ABI's refusals before any CUDA call."""
import ctypes
import json
import os
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import bert_ref
from oracle import mpnet_ref
from ragmeup_b200.weights import PRESETS, MPNetConfig, synthetic_bert_weights, weight_names

GOLDEN = [("all-mpnet-base-v2", 0, 1.0), ("tiny-mpnet", 2, 4.0)]
LOG2E = np.float32(1.4426950408889634)


def _cfg(preset):
    return MPNetConfig(**asdict(PRESETS[preset][0]))


@pytest.mark.parametrize("preset,seed,scale", GOLDEN)
def test_mpnet_oracle_matches_hf(golden_dir, preset, seed, scale):
    """the fp32 forward (padded, pad id 1) and the float64 ragged stack both match MPNetModel at BERT's bar"""
    g = np.load(f"{golden_dir}/mpnet.npz")
    key = f"mpnet_{preset}_{seed}_{scale}"
    cfg = _cfg(preset)
    ocfg = mpnet_ref.MPNetCfg(**asdict(cfg))
    w = synthetic_bert_weights(cfg, seed=seed, with_head=False, scale=scale)
    ids = torch.from_numpy(g[key + "_ids"].astype(np.int64))
    mask = torch.from_numpy(g[key + "_mask"].astype(np.int64))
    assert (ids == 1).logical_and(mask == 1).any(), "the goldens hold a literal id 1 inside a text"
    lens = mask.sum(1).tolist()
    with torch.no_grad():
        h = mpnet_ref.mpnet_encoder_forward(w, ocfg, ids, mask)
        mean = bert_ref.l2_normalize(bert_ref.pool(h, mask, "mean")).numpy()
        cls = bert_ref.l2_normalize(bert_ref.pool(h, mask, "cls")).numpy()
    h_last = np.stack([h[b, n - 1].numpy() for b, n in enumerate(lens)])
    tol = 4e-6 if scale == 1.0 else 2e-5
    assert np.abs(mean - g[key + "_mean"]).max() < tol
    assert np.abs(cls - g[key + "_cls"]).max() < tol
    assert np.abs(h[:, 0].numpy() - g[key + "_h_first"]).max() < 50 * tol
    assert np.abs(h_last - g[key + "_h_last"]).max() < 50 * tol
    # the float64 reference of the kernels, on the ragged batch
    flat = np.concatenate([g[key + "_ids"][b, :n] for b, n in enumerate(lens)])
    cu = np.r_[0, np.cumsum(lens)]
    ref = mpnet_ref.mpnet_stack_ref(w, cfg, flat, cu)
    assert float((ref["mean_norm"] - torch.from_numpy(g[key + "_mean"]).double()).abs().max()) < tol
    assert float((ref["cls_norm"] - torch.from_numpy(g[key + "_cls"]).double()).abs().max()) < tol
    assert float((ref["hidden"][cu[1:] - 1] - torch.from_numpy(g[key + "_h_last"]).double()).abs().max()) < 50 * tol


def test_bias_table_follows_transformers_buckets():
    """rmu_relative_bias_table (what rmu_encoder_create builds, host only) with bias[b, h] = b + 32 h: entry
    clamp(rel, -127, 127) + 127 of head h is (bucket(rel) + 32 h) log2(e) for every rel in [-1023, 1023]"""
    from transformers.models.mpnet.modeling_mpnet import MPNetEncoder
    from ragmeup_b200 import _lib
    rel = np.arange(-1023, 1024)
    want = MPNetEncoder.relative_position_bucket(torch.from_numpy(rel)).numpy()
    assert np.array_equal(mpnet_ref.relative_position_bucket(rel), want)
    heads = 3
    bias = (np.arange(32)[:, None] + 32 * np.arange(heads)[None, :]).astype(np.float32)
    tab = np.zeros((heads, 255), np.float32)
    assert _lib.lib().rmu_relative_bias_table(bias.ctypes.data, 32, heads, tab.ctypes.data) == 0
    idx = np.clip(rel, -127, 127) + 127
    for h in range(heads):
        assert np.array_equal(tab[h, idx], (want + 32 * h).astype(np.float32) * LOG2E), h
    assert np.allclose(mpnet_ref.bias_table(bias, heads).numpy(), tab, rtol=2 ** -23, atol=0)
    assert _lib.lib().rmu_relative_bias_table(bias.ctypes.data, 16, heads, tab.ctypes.data) == -3
    assert _lib.lib().rmu_relative_bias_table(None, 32, heads, tab.ctypes.data) == -1


def test_position_ids_rule():
    ids = torch.tensor([[0, 7, 1, 9, 1, 1, 4, 2], [1, 1, 5, 2, 1, 1, 1, 1]])
    assert mpnet_ref.position_ids(ids).tolist() == [[2, 3, 1, 4, 1, 1, 5, 6], [1, 1, 2, 3, 1, 1, 1, 1]]


def _mpnet_snapshot(root, name, cfg, prefix="", buckets=32, extra=None):
    """an MPNet snapshot in transformers' naming (optionally under `mpnet.`), sentence-transformers modules included"""
    from safetensors.numpy import save_file
    path = os.path.join(root, name)
    os.makedirs(os.path.join(path, "1_Pooling"), exist_ok=True)
    w = synthetic_bert_weights(cfg, seed=5, with_head=False)
    inv = (("attention.self.query.", "attention.attn.q."), ("attention.self.key.", "attention.attn.k."),
           ("attention.self.value.", "attention.attn.v."), ("attention.output.dense.", "attention.attn.o."),
           ("attention.output.LayerNorm.", "attention.LayerNorm."))
    sd = {}
    for k, v in w.items():
        if k == "embeddings.token_type_embeddings.weight":
            continue
        if k == mpnet_ref.REL_BIAS and buckets != 32:
            v = np.concatenate([v, np.full((buckets - 32, cfg.heads), 9.0, np.float32)])[:buckets]
        for a, b in inv:
            k = k.replace(a, b)
        sd[prefix + k] = v
    sd[prefix + "pooler.dense.weight"] = np.zeros((cfg.hidden, cfg.hidden), np.float32)
    save_file(sd, os.path.join(path, "model.safetensors"))
    conf = {"model_type": "mpnet", "vocab_size": cfg.vocab_size, "hidden_size": cfg.hidden,
            "num_hidden_layers": cfg.layers, "num_attention_heads": cfg.heads, "intermediate_size": cfg.ffn,
            "max_position_embeddings": cfg.max_pos, "layer_norm_eps": 1e-5, "hidden_act": "gelu",
            "relative_attention_num_buckets": buckets, **(extra or {})}
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(conf, f)
    with open(os.path.join(path, "modules.json"), "w") as f:
        json.dump([{"path": "", "type": "sentence_transformers.models.Transformer"},
                   {"path": "1_Pooling", "type": "sentence_transformers.models.Pooling"},
                   {"path": "2_Normalize", "type": "sentence_transformers.models.Normalize"}], f)
    with open(os.path.join(path, "1_Pooling", "config.json"), "w") as f:
        json.dump({"pooling_mode_mean_tokens": True}, f)
    return path, w


@pytest.mark.parametrize("prefix,buckets", [("", 32), ("mpnet.", 32), ("", 64)])
def test_snapshot_resolution(tmp_path, prefix, buckets):
    from ragmeup_b200.weights import resolve_model
    cfg = _cfg("tiny-mpnet")
    path, w = _mpnet_snapshot(str(tmp_path), "m", cfg, prefix, buckets)
    got_cfg, got, pooling, normalize, max_len, _act, src = resolve_model(path, with_head=False)
    assert isinstance(got_cfg, MPNetConfig) and (got_cfg.position_mode, got_cfg.rel_buckets) == (1, 32)
    assert got_cfg.ln_eps == 1e-5 and got_cfg.type_vocab == 1
    assert (pooling, normalize, max_len, src) == ("mean", True, cfg.max_pos - 2, path)
    for name, shape in weight_names(got_cfg, False):
        assert got[name].shape == shape, name
        if name == "embeddings.token_type_embeddings.weight":
            assert not got[name].any()
        else:
            assert np.array_equal(got[name], w[name]), name        # rows 0..31 of a larger bias table


def test_refusals(tmp_path):
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.flashrank import Ranker
    from ragmeup_b200.weights import resolve_model
    cfg = _cfg("tiny-mpnet")
    path, _ = _mpnet_snapshot(str(tmp_path), "few", cfg, buckets=32, extra={"relative_attention_num_buckets": 16})
    with pytest.raises(ValueError, match="relative_attention_num_buckets"):
        resolve_model(path, with_head=False)
    path, _ = _mpnet_snapshot(str(tmp_path), "ms-marco-MiniLM-L-12-v2", cfg)
    for make in (lambda: HuggingFaceCrossEncoder(model_name=path), lambda: HuggingFaceCrossEncoder("synthetic:tiny-mpnet"),
                 lambda: Ranker("ms-marco-MiniLM-L-12-v2", cache_dir=str(tmp_path)), lambda: Ranker("synthetic:tiny-mpnet")):
        with pytest.raises(ValueError, match="MPNet"):
            make()
    r = resolve_model("synthetic:multi-qa-mpnet-base-dot-v1", with_head=False)
    assert (r[2], r[3], r[4]) == ("cls", False, 512)
    r = resolve_model("synthetic:all-mpnet-base-v2", with_head=False)
    assert (r[0].hidden, r[0].layers, r[0].heads, r[0].ffn, r[0].max_pos, r[2], r[3], r[4]) == \
        (768, 12, 12, 3072, 514, "mean", True, 384)
    assert _cfg("tiny-mpnet").head_dim == 32


def test_synthetic_tokenizer_templates():
    from ragmeup_b200.tokenizer import RaggedTokenizer, load_tokenizer, synthetic_mpnet_vocab, synthetic_vocab
    tok = load_tokenizer(None, 30527, mpnet=True)
    v = synthetic_mpnet_vocab(30527)
    assert [v[t] for t in ("<s>", "<pad>", "</s>", "<unk>", "[UNK]", "<mask>")] == [0, 1, 2, 3, 104, 30526]
    assert len(v) == 30527 and sorted(v.values()) == list(range(30527))
    e = tok.encode("ba ce")
    assert e.ids[0] == 0 and e.ids[-1] == 2 and not any(e.type_ids)
    p = tok.encode("ba", "ce")
    assert p.ids == [0, v["ba"], 2, 2, v["ce"], 2] and not any(p.type_ids)
    # the literal "<pad>" is the special token, id 1, with attention mask 1
    e = tok.encode("ba <pad> ce")
    assert e.ids == [0, v["ba"], 1, v["ce"], 2] and e.attention_mask == [1] * 5
    ids, typ, cu = RaggedTokenizer(tok, 4)(["<pad>", "ba ce di fo"])
    assert ids.tolist() == [0, 1, 2, 0, v["ba"], v["ce"], 2] and cu.tolist() == [0, 3, 7] and not typ.any()
    # the BERT synthetic vocabulary is unchanged
    assert synthetic_vocab(30522)["[CLS]"] == 101 and load_tokenizer(None, 30522).encode("<pad>").ids[0] == 101


def _create(cfg, arrs, has_head=0):
    from ragmeup_b200 import _lib
    ptrs = (ctypes.c_void_p * len(arrs))(*[None if a is None else a.ctypes.data for a in arrs])
    cc = _lib.BertConfigC(cfg.vocab_size, cfg.hidden, cfg.layers, cfg.heads, cfg.ffn, cfg.max_pos, cfg.type_vocab,
                          cfg.num_labels, cfg.ln_eps, cfg.position_mode, cfg.rel_buckets)
    h = ctypes.c_void_p()
    rc = _lib.lib().rmu_encoder_create(ctypes.byref(cc), ptrs, len(arrs), has_head, ctypes.byref(h))
    if rc == 0:
        _lib.lib().rmu_encoder_destroy(h)
    return rc


def test_abi_refusals_before_any_cuda_call():
    from ragmeup_b200 import _lib
    l = _lib.lib()
    cfg = _cfg("tiny-mpnet")
    w = synthetic_bert_weights(cfg, seed=0, with_head=False)
    arrs = [np.ascontiguousarray(w[n]) for n, _ in weight_names(cfg, False)]
    for kw in (dict(rel_buckets=16), dict(rel_buckets=64), dict(position_mode=2), dict(position_mode=-1)):
        assert _create(MPNetConfig(**{**asdict(cfg), **kw}), arrs) == -3, kw
    assert _create(cfg, arrs[:-1]) == -1                           # the bias table missing
    assert _create(cfg, arrs[:-1] + [None]) == -1                  # a null bias table
    assert _create(MPNetConfig(**{**asdict(cfg), "rel_buckets": 0}), arrs) == -1   # one tensor too many
    assert _create(cfg, arrs) in (0, -2)                           # accepted: without a device the next step fails
    p = 1 << 20
    att = lambda **k: l.rmu_debug_attention_bias(  # noqa: E731
        p, p, k.get("cq", None), k.get("cl", None), p, k.get("B", 2), k.get("H", 128), k.get("heads", 4), 16,
        k.get("tab", p), p, p, None)
    assert att(tab=None) == -1
    assert att(cq=p) == -1                                         # one compact Q plane without the other
    assert att(B=0) == -1
    assert att(heads=8) == -3                                      # d_h = 16
    emb = lambda mode, H=128: l.rmu_debug_embed_ln_pos(p, None, p, 1, 4, H, 100, 16, 1, p, p, p, p, p, 1e-5, mode, p, p,  # noqa: E731
                                                      None)
    assert emb(2) == -1 and emb(-1) == -1 and emb(1, H=100) == -3
