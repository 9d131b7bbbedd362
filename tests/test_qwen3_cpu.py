"""Qwen3 on the host: config forms and refusals, bf16 and sharded snapshots, the float64 oracle against transformers,
the goldens, tokenisation and the reranker's prompt, and the C entry point's refusals (before any CUDA call)."""
from __future__ import annotations

import ctypes as C
import importlib.util
import json
import os
from dataclasses import asdict, replace

import numpy as np
import pytest
import torch

from oracle import qwen3_ref as qr
from ragmeup_b200.weights import (PRESETS, QWEN3_RERANK_INSTRUCTION, QWEN3_RERANK_PREFIX, QWEN3_RERANK_SUFFIX,
                                  Qwen3Config, load_hf_snapshot, qwen3_weight_names, resolve_colbert, resolve_model,
                                  synthetic_qwen3_weights)

HF5 = {"model_type": "qwen3", "vocab_size": 151669, "hidden_size": 1024, "intermediate_size": 3072,
       "num_hidden_layers": 28, "num_attention_heads": 16, "num_key_value_heads": 8, "head_dim": 128,
       "max_position_embeddings": 40960, "rms_norm_eps": 1e-6, "hidden_act": "silu", "attention_bias": False,
       "use_sliding_window": False, "layer_types": ["full_attention"] * 28, "tie_word_embeddings": True,
       "rope_parameters": {"rope_type": "default", "rope_theta": 1000000.0}, "pad_token_id": None}


def _golden_module():
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden_qwen3.py")
    spec = importlib.util.spec_from_file_location("make_golden_qwen3", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_config_forms():
    cfg = Qwen3Config.from_hf(HF5)
    assert (cfg.hidden, cfg.heads, cfg.kv_heads, cfg.head_dim, cfg.ffn, cfg.layers) == (1024, 16, 8, 128, 3072, 28)
    assert cfg.rope_theta == 1e6 and cfg.tie_word_embeddings and cfg.pad_token_id is None and cfg.head_pad_id == -1
    old = {k: v for k, v in HF5.items() if k not in ("rope_parameters", "layer_types")}
    old.update(rope_theta=500000.0, rope_scaling=None, pad_token_id=151643, num_labels=1)
    cfg = Qwen3Config.from_hf(old)
    assert cfg.rope_theta == 500000.0 and cfg.head_pad_id == 151643
    assert replace(cfg, reranker=True).head_pad_id == -1


def test_transformers_config_round_trip():
    transformers = pytest.importorskip("transformers")
    d = transformers.Qwen3Config(**{k: v for k, v in HF5.items() if k != "model_type"}).to_dict()
    cfg = Qwen3Config.from_hf(d)
    assert (cfg.kv_heads, cfg.head_dim, cfg.rope_theta, cfg.ln_eps) == (8, 128, 1e6, 1e-6)


@pytest.mark.parametrize("field,value", [("hidden_act", "gelu"), ("attention_bias", True), ("use_sliding_window", True),
                                         ("layer_types", ["full_attention"] * 27 + ["sliding_attention"]),
                                         ("rope_scaling", {"rope_type": "yarn", "factor": 4.0}),
                                         ("rope_parameters", {"rope_type": "yarn", "rope_theta": 1e6}),
                                         ("model_type", "qwen3_moe")])
def test_refusals_name_the_field(field, value):
    d = dict(HF5, **{field: value})
    name = "rope_type" if field == "rope_parameters" else field
    with pytest.raises(ValueError, match=name):
        Qwen3Config.from_hf(d)


@pytest.mark.parametrize("kind", ["qwen3_moe", "qwen2"])
def test_other_qwen_model_types_are_refused(tmp_path, kind):
    (tmp_path / "config.json").write_text(json.dumps(dict(HF5, model_type=kind)))
    with pytest.raises(ValueError, match=kind):
        load_hf_snapshot(str(tmp_path), with_head=False)


@pytest.fixture(scope="module")
def golden_setup():
    pytest.importorskip("transformers")
    mod = _golden_module()
    cfg, w, lm, tok = mod.build()
    return mod, cfg, w, lm, tok


@pytest.fixture(scope="module")
def snapshots(golden_setup, tmp_path_factory):
    mod, cfg, w, lm, tok = golden_setup
    return mod.save_snapshots(str(tmp_path_factory.mktemp("qwen3")), cfg, w, lm, tok)


def test_snapshot_without_tokenizer_json_is_refused(snapshots, tmp_path):
    import shutil
    d = tmp_path / "s"
    shutil.copytree(snapshots["seqcls"], d)
    os.remove(d / "tokenizer.json")
    with pytest.raises(ValueError, match="tokenizer.json"):
        load_hf_snapshot(str(d), with_head=True)


def test_snapshot_pooling_other_than_lasttoken_is_refused(snapshots, tmp_path):
    import shutil
    d = tmp_path / "s"
    shutil.copytree(snapshots["embedder"], d)
    (d / "1_Pooling" / "config.json").write_text(json.dumps({"pooling_mode_mean_tokens": True}))
    with pytest.raises(ValueError, match="last token"):
        load_hf_snapshot(str(d), with_head=False)


def test_seqcls_without_pad_token_id_is_refused(snapshots, tmp_path):
    import shutil
    d = tmp_path / "s"
    shutil.copytree(snapshots["seqcls"], d)
    cfgd = json.loads((d / "config.json").read_text())
    cfgd["pad_token_id"] = None
    (d / "config.json").write_text(json.dumps(cfgd))
    with pytest.raises(ValueError, match="pad_token_id"):
        load_hf_snapshot(str(d), with_head=True)


def test_snapshot_forms_and_heads(golden_setup, snapshots):
    mod, cfg, w, lm, tok = golden_setup
    c, we, pooling, normalize, max_len, act = load_hf_snapshot(snapshots["embedder"], with_head=False)
    assert (pooling, normalize, max_len, act, c.prompt) == ("last", True, 1024, "identity", "")
    assert set(we) == {n for n, _ in qwen3_weight_names(c, False)}
    c, ws, *_rest, act = load_hf_snapshot(snapshots["seqcls"], with_head=True)
    assert act == "sigmoid" and c.head_pad_id == tok.token_to_id("<|endoftext|>") and np.array_equal(ws["head"], w["head"])
    c, wr, *_rest, act = load_hf_snapshot(snapshots["reranker"], with_head=True)
    yes, no = tok.token_to_id("yes"), tok.token_to_id("no")
    assert act == "yes_prob" and c.reranker and c.num_labels == 2 and np.array_equal(wr["head"], lm[[no, yes]])
    assert resolve_colbert(snapshots["reranker"]) is None


def test_default_prompt_is_applied_only_when_set(snapshots, tmp_path):
    import shutil
    d = tmp_path / "s"
    shutil.copytree(snapshots["embedder"], d)
    (d / "config_sentence_transformers.json").write_text(json.dumps({"prompts": {"query": "Instruct: x\nQuery:"},
                                                                      "default_prompt_name": None}))
    assert load_hf_snapshot(str(d), with_head=False)[0].prompt == ""
    (d / "config_sentence_transformers.json").write_text(json.dumps({"prompts": {"query": "Instruct: x\nQuery:"},
                                                                      "default_prompt_name": "query"}))
    assert load_hf_snapshot(str(d), with_head=False)[0].prompt == "Instruct: x\nQuery:"


def test_bf16_and_sharded_snapshots_load_as_fp32(golden_setup, snapshots, tmp_path):
    """a bfloat16 save loads to the float32 widening of the bf16 weights; a sharded save to the same arrays as one file"""
    import transformers
    mod, cfg, w, lm, tok = golden_setup
    _c, w32, *_ = load_hf_snapshot(snapshots["seqcls"], with_head=True)
    bdirs = mod.save_snapshots(str(tmp_path / "bf16"), cfg, w, lm, tok, bf16=True)
    _c, wb, *_ = load_hf_snapshot(bdirs["seqcls"], with_head=True)
    for k, v in w32.items():
        assert wb[k].dtype == np.float32
        assert np.array_equal(wb[k], torch.from_numpy(v).to(torch.bfloat16).float().numpy()), k
    sh = tmp_path / "sharded"
    m = transformers.Qwen3ForSequenceClassification.from_pretrained(snapshots["seqcls"])
    m.save_pretrained(sh, safe_serialization=True, max_shard_size="300KB")
    tok.save(str(sh / "tokenizer.json"))
    assert not (sh / "model.safetensors").exists() and (sh / "model.safetensors.index.json").exists()
    _c, ws, *_ = load_hf_snapshot(str(sh), with_head=True)
    assert set(ws) == set(w32) and all(np.array_equal(ws[k], w32[k]) for k in w32)
    rdir = tmp_path / "rr"
    transformers.Qwen3ForCausalLM.from_pretrained(snapshots["reranker"]).save_pretrained(
        rdir, safe_serialization=True, max_shard_size="300KB")
    tok.save(str(rdir / "tokenizer.json"))
    _c, wr, *_ = load_hf_snapshot(str(rdir), with_head=True)
    assert np.array_equal(wr["head"], lm[[tok.token_to_id("no"), tok.token_to_id("yes")]])


def test_oracle_matches_transformers_float64(golden_setup, monkeypatch):
    """the float64 oracle against transformers' three models in float64: |delta| <= 1e-10.  Two of transformers' steps
    run in float32 whatever the model's dtype, and are kept in float64 here: eager attention's softmax (so sdpa), and
    Qwen3RMSNorm's upcast to float32 (its formula, w * (x * rsqrt(mean(x^2) + eps)), in the input's dtype)"""
    from transformers.models.qwen3 import modeling_qwen3
    mod, cfg, w, lm, tok = golden_setup

    def rms64(self, x):
        return self.weight * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.variance_epsilon))
    monkeypatch.setattr(modeling_qwen3.Qwen3RMSNorm, "forward", rms64)
    base, seq, lmm = (m.double() for m in mod.hf_models(cfg, w, lm, attn="sdpa"))
    seqs = [e.ids for e in tok.encode_batch(mod.texts(3, 1, 90, 50))]
    W = qr.weights(w)
    yes, no = tok.token_to_id("yes"), tok.token_to_id("no")
    with torch.no_grad():
        for s in seqs:
            x = torch.tensor([s])
            h = qr.hidden(W, cfg, s)
            assert float((h - base(x).last_hidden_state[0]).abs().max()) <= 1e-10
            want = seq(x).logits[0]
            assert float((qr.logits(W, cfg, [s], cfg.head_pad_id)[0] - want).abs().max()) <= 1e-10
            lg = lmm(x).logits[0, -1]
            mine = qr.yes_probability((h[-1] @ torch.from_numpy(lm[[no, yes]]).double().T)[None])[0]
            assert abs(float(mine) - float(torch.stack([lg[no], lg[yes]]).log_softmax(0)[1].exp())) <= 1e-10


def test_oracle_matches_goldens(golden_setup, golden_dir):
    mod, cfg, w, lm, tok = golden_setup
    g = np.load(os.path.join(golden_dir, "qwen3.npz"))
    split = lambda ids, cu: [ids[cu[b]:cu[b + 1]].tolist() for b in range(len(cu) - 1)]   # noqa: E731
    body = {k: v for k, v in w.items() if k != "head"}
    emb = qr.embed(body, cfg, split(g["emb_ids"], g["emb_cu"]), True, torch.float32).numpy()
    assert np.abs(emb - g["emb"]).max() < 1e-5
    lg = qr.logits(w, cfg, split(g["cls_ids"], g["cls_cu"]), cfg.head_pad_id, torch.float32).numpy()
    assert np.abs(lg - g["cls_logits"]).max() < 1e-5
    yes, no = (int(i) for i in g["yes_no"])
    rr = qr.yes_probability(qr.logits({**body, "head": lm[[no, yes]]}, cfg, split(g["rr_ids"], g["rr_cu"]), -1,
                                      torch.float32)).numpy()
    assert np.abs(rr - g["rr_scores"]).max() < 1e-5


def test_golden_script_reproduces_the_fixture(golden_setup, golden_dir):
    mod = golden_setup[0]
    g = np.load(os.path.join(golden_dir, "qwen3.npz"))
    with torch.no_grad():
        new = mod.compute()
    assert set(new) == set(g.files)
    for k in g.files:
        assert new[k].dtype == g[k].dtype and np.array_equal(new[k], g[k]), k


def test_tokenisation_and_reranker_prompt_equal_transformers(golden_setup, snapshots):
    """the embedder's texts, the sequence-classification pairs and the reranker's prompt, against the same tokenizer
    through transformers (PreTrainedTokenizerFast) and the model card's process_inputs"""
    from transformers import PreTrainedTokenizerFast
    from ragmeup_b200.cross_encoder import Qwen3RerankPrompt
    from ragmeup_b200.tokenizer import RaggedTokenizer, load_tokenizer
    mod, cfg, w, lm, tok = golden_setup
    hf = PreTrainedTokenizerFast(tokenizer_object=tok)
    t = load_tokenizer(snapshots["embedder"], qwen3=True)
    texts = mod.texts(8, 1, 400, 60)
    for L in (64, 1024):
        ids, _typ, cu = RaggedTokenizer(t, L)(texts)
        want = hf(texts, truncation=True, max_length=L)["input_ids"]
        assert [ids[cu[b]:cu[b + 1]].tolist() for b in range(len(texts))] == want
        assert all(s[-1] == tok.token_to_id("<|endoftext|>") for s in want)
    qs, ds = mod.texts(4, 2, 30, 61), mod.texts(4, 5, 300, 62)
    ids, _typ, cu = RaggedTokenizer(t, 96)(qs, ds)
    want = hf(qs, ds, truncation="longest_first", max_length=96)["input_ids"]
    assert [ids[cu[b]:cu[b + 1]].tolist() for b in range(len(qs))] == want
    fixed = len(Qwen3RerankPrompt(t, 8192).prefix) + len(Qwen3RerankPrompt(t, 8192).suffix)
    for L in (fixed + 40, 8192):                   # the first truncates the formatted text
        p = Qwen3RerankPrompt(t, L)
        ids, typ, cu = p(qs, ds)
        assert typ is None
        want = qr.rerank_ids(hf, QWEN3_RERANK_PREFIX, QWEN3_RERANK_SUFFIX, QWEN3_RERANK_INSTRUCTION, list(zip(qs, ds)), L)
        assert [ids[cu[b]:cu[b + 1]].tolist() for b in range(len(qs))] == want
        assert max(np.diff(cu)) <= L
    assert len(Qwen3RerankPrompt(t, 8192).prefix) > 5 and tok.token_to_id("<|im_start|>") in Qwen3RerankPrompt(t, 8192).prefix


def test_presets_resolve():
    cfg, w, pooling, normalize, max_len, act, src = resolve_model("synthetic:tiny-qwen3", with_head=False)
    assert isinstance(cfg, Qwen3Config) and pooling == "last" and normalize and src is None
    assert cfg.head_dim == 128 and cfg.kv_heads < cfg.heads and cfg.layers >= 3 and cfg.name == "synthetic:tiny-qwen3"
    assert set(w) == {n for n, _ in qwen3_weight_names(cfg, False)}
    cfg, w, *_r, act, _s = resolve_model("synthetic:tiny-qwen3", with_head=True)
    assert act == "sigmoid" and w["head"].shape == (1, cfg.hidden)
    cfg = PRESETS["qwen3-reranker-0.6b"][0]
    assert cfg.reranker and cfg.num_labels == 2 and (cfg.hidden, cfg.kv_heads, cfg.ffn) == (1024, 8, 3072)


def test_flashrank_and_colbert_refuse_qwen3():
    from ragmeup_b200.weights import load_colbert_snapshot, resolve_flashrank
    with pytest.raises(ValueError, match="Qwen3"):
        resolve_flashrank("synthetic:tiny-qwen3")
    assert resolve_colbert("synthetic:tiny-qwen3") is None


def test_colbert_loader_refuses_qwen3(tmp_path):
    from ragmeup_b200.weights import load_colbert_snapshot
    (tmp_path / "config.json").write_text(json.dumps(HF5))
    with pytest.raises(ValueError, match="qwen3"):
        load_colbert_snapshot(str(tmp_path))


def _create(cfg, kv=None, head_dim=128, rope_rows=None, rope_half=64, head_form=0, has_head=0, n=None, nulls=(),
            arrays=None):
    from ragmeup_b200 import _lib
    qx = _lib.Qwen3ExtC(cfg.kv_heads if kv is None else kv, head_dim, cfg.max_pos if rope_rows is None else rope_rows,
                        rope_half, head_form, -1)
    count = 1 + 11 * cfg.layers + 1 + has_head + 2 if n is None else n
    dummy = np.zeros(1, np.float32)
    ptrs = (C.c_void_p * count)(*[None if i in nulls else (arrays[i].ctypes.data if arrays else dummy.ctypes.data)
                                  for i in range(count)])
    h = C.c_void_p()
    cc = _lib.bert_config_c(cfg)
    return _lib.lib().rmu_encoder_create_qwen3(C.byref(cc), C.byref(qx), ptrs, count, has_head, C.byref(h))


def test_c_refusals_before_any_cuda_call():
    """every refusal returns before a CUDA call (the tensors are 1-element dummies; the machine may have no GPU)"""
    from ragmeup_b200 import _lib
    ERR_ARG, UNSUP = -1, -3
    cfg = Qwen3Config(**asdict(PRESETS["tiny-qwen3"][0]))
    assert _create(cfg, head_dim=64) == UNSUP
    assert _create(replace(cfg, hidden=200)) == UNSUP                          # H % 128
    assert _create(replace(cfg, hidden=4224)) == UNSUP                         # H > 4096
    assert _create(replace(cfg, ffn=400)) == UNSUP                             # F % 64
    assert _create(cfg, kv=3) == UNSUP                                         # heads % kv_heads
    assert "num_key_value_heads" in _lib.lib().rmu_last_error().decode()
    assert _create(cfg, kv=0) == UNSUP
    assert _create(cfg, rope_rows=cfg.max_pos - 1) == ERR_ARG
    assert _create(cfg, rope_half=128) == ERR_ARG
    assert _create(cfg, head_form=1) == ERR_ARG                                # a head form without a head
    assert _create(cfg, has_head=1) == ERR_ARG                                 # a head without its form
    assert _create(cfg, n=1 + 11 * cfg.layers + 1 + 1) == ERR_ARG             # a rope table missing
    assert _create(cfg, nulls=(3,)) == ERR_ARG

    class WithRel(Qwen3Config):
        rel_buckets = 32
    assert _create(WithRel(**asdict(cfg))) == UNSUP
    # a GEMM weight outside the split planes' range, found on the host before any CUDA call
    from ragmeup_b200.weights import rope_table
    w = synthetic_qwen3_weights(cfg, 0)
    w["layers.1.mlp.up_proj.weight"][3, 5] = 70000.0
    arrays = [np.ascontiguousarray(w[n]) for n, _ in qwen3_weight_names(cfg, False)]
    arrays += list(rope_table(cfg.rope_theta, cfg.head_dim, cfg.max_pos))
    assert _create(cfg, arrays=arrays) == UNSUP
    assert "layer 1 up_proj" in _lib.lib().rmu_last_error().decode()
