"""CPU: 70B-class decoders in NF4 built layer by layer.  The C refusals of rmu_decoder_create_nf4 and
rmu_decoder_load_layer_nf4 that come before any CUDA call, the split-weight refusal above hidden 4096, the device-memory
plan against the sizes computed from the published shapes, the per-layer snapshot reader against the whole-snapshot
loader, and the rule that frees the reference's own transformers copy of the model."""
import ctypes as C
import json
import os
from dataclasses import replace

import numpy as np
import pytest

from ragmeup_b200 import _lib
from ragmeup_b200.weights import (DECODER_PRESETS, LlamaConfig, Qwen3Config, _load_decoder_snapshot, check_decoder_plan,
                                  decoder_config, decoder_layers, decoder_memory_plan, resolve_decoder)

ERR_ARG, UNSUP = -1, -3


def _create(cfg, qk=0, hd=128, kv=None, rope_rows=None, head_form=0):
    p = 1 << 20                                     # stand-in host addresses: a refusal never reads them
    cc = _lib.bert_config_c(cfg)
    qx = _lib.Qwen3ExtC(cfg.kv_heads if kv is None else kv, hd, cfg.max_pos if rope_rows is None else rope_rows, 64,
                        head_form, -1)
    h = C.c_void_p()
    rc = _lib.lib().rmu_decoder_create_nf4(C.byref(cc), C.byref(qx), qk, p, p, p, p, C.byref(h))
    assert not h.value
    return rc


def test_create_refusals_before_any_cuda_call():
    big = decoder_config("synthetic:llama-3.1-70b")
    l = _lib.lib()
    assert _create(replace(big, hidden=8320, heads=65)) == UNSUP                      # above 8192
    assert b"up to 8192, got 8320" in l.rmu_last_error()
    assert _create(replace(big, hidden=8192 - 64)) == UNSUP                           # not a multiple of 128
    assert _create(big, hd=64) == UNSUP and b"head_dim must be 128" in l.rmu_last_error()
    assert _create(replace(big, ffn=28672 + 32)) == UNSUP                             # F % 64
    assert _create(big, kv=7) == UNSUP                                                # 64 heads over 7 kv heads
    assert _create(big, rope_rows=big.max_pos - 1) == ERR_ARG
    assert _create(big, head_form=1) == ERR_ARG                                       # decoders have no head
    assert _create(replace(big, ffn=49152 + 64)) == UNSUP                             # down's K above the GEMV's
    assert b"49152" in l.rmu_last_error()
    assert _create(big, qk=2) == ERR_ARG
    cc, qx, h = _lib.bert_config_c(big), _lib.Qwen3ExtC(8, 128, big.max_pos, 64, 0, -1), C.c_void_p()
    assert l.rmu_decoder_create_nf4(C.byref(cc), C.byref(qx), 0, None, 1, 1, 1, C.byref(h)) == ERR_ARG
    assert l.rmu_decoder_create_nf4(None, C.byref(qx), 0, 1, 1, 1, 1, C.byref(h)) == ERR_ARG
    ptrs = (C.c_void_p * 9)(*([1 << 20] * 9))
    assert l.rmu_decoder_load_layer_nf4(None, 0, ptrs, None) == ERR_ARG
    # split handles keep their limit of 4096
    small = LlamaConfig(**{**DECODER_PRESETS["tiny-llama"].__dict__, "hidden": 4224, "heads": 33})
    arrs = [np.zeros(1, np.float32)] * (1 + 9 * small.layers + 1 + 2)
    pp = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    cc, qx = _lib.bert_config_c(small), _lib.Qwen3ExtC(small.kv_heads, 128, small.max_pos, 64, 0, -1)
    assert l.rmu_encoder_create_llama(C.byref(cc), C.byref(qx), pp, len(arrs), C.byref(h)) == UNSUP
    assert b"up to 4096" in l.rmu_last_error()


def test_split_weights_above_4096_are_refused_naming_the_setting():
    from ragmeup_b200 import provenance
    for name in ("synthetic:llama-3.1-70b", "synthetic:qwen3-32b"):
        with pytest.raises(ValueError, match=r"RMU_DECODER_WEIGHTS=nf4") as e:
            provenance.DecoderAttention(name, weights="split")
        assert str(decoder_memory_plan(decoder_config(name), "split")["total"]) in str(e.value)
    check_decoder_plan(decoder_config("synthetic:llama-3.1-8b"), "split")            # 4096 still takes split planes


def test_memory_plan_matches_the_computed_sizes():
    """GB = 1e9 bytes, rounded to 0.1 as the table in INTEGRATION.md states them"""
    def gb(v):
        return round(v / 1e9, 1)
    want = {  # layers (NF4 codes + absmax), fp32 embeddings, LM head planes, prefill scratch, total
        "llama-3.1-8b": (3.9, 2.1, 2.1, 0.5, 8.7),
        "llama-3.1-70b": (38.5, 4.2, 4.2, 1.9, 48.9),
        "qwen3-32b": (17.6, 3.1, 3.1, 1.0, 24.8),
    }
    for preset, (layers, emb, head, scratch, total) in want.items():
        cfg = decoder_config("synthetic:" + preset)
        plan = decoder_memory_plan(cfg, "nf4")
        assert (gb(plan["layers"]), gb(plan["embeddings"]), gb(plan["lm_head"]), gb(plan["scratch"]),
                gb(plan["total"])) == (layers, emb, head, scratch, total), preset
        assert plan["build_peak"] == plan["total"] + (1 << 24) * 6
    big = decoder_config("synthetic:llama-3.1-70b")
    QD, KD = 64 * 128, 8 * 128
    per_layer = (QD + 2 * KD) * 8192 + 8192 * QD + 2 * 28672 * 8192 + 8192 * 28672
    assert per_layer == 855_638_016
    assert decoder_memory_plan(big, "nf4")["layers"] == 80 * per_layer * 9 // 16
    assert decoder_memory_plan(big, "split")["layers"] == 80 * per_layer * 4
    with pytest.raises(ValueError, match=r"48961934336 bytes .*RMU_DECODER_WEIGHTS=nf4.* 40000000000 bytes"):
        check_decoder_plan(big, "nf4", free_bytes=40_000_000_000)
    check_decoder_plan(big, "nf4", free_bytes=79_000_000_000)


def test_presets_are_the_published_shapes():
    l70 = decoder_config("synthetic:llama-3.1-70b")
    assert isinstance(l70, LlamaConfig)
    assert (l70.vocab_size, l70.hidden, l70.layers, l70.heads, l70.kv_heads, l70.ffn, l70.max_pos, l70.rope_theta,
            l70.rope_scaling) == (128256, 8192, 80, 64, 8, 28672, 131072, 500000.0, (8.0, 1.0, 4.0, 8192))
    q32 = decoder_config("synthetic:qwen3-32b")
    assert isinstance(q32, Qwen3Config) and q32.name == "synthetic:qwen3-32b" and q32.num_labels == 1
    assert (q32.vocab_size, q32.hidden, q32.layers, q32.heads, q32.kv_heads, q32.ffn, q32.max_pos, q32.rope_theta,
            q32.ln_eps, q32.tie_word_embeddings) == (151936, 5120, 64, 64, 8, 25600, 40960, 1e6, 1e-6, False)


@pytest.mark.parametrize("name", ["synthetic:tiny-llama:3:2.0", "synthetic:tiny-qwen3:1"])
def test_synthetic_layers_are_the_whole_draw(name):
    cfg, w = resolve_decoder(name)
    src = decoder_layers(name)
    assert src.cfg == cfg
    g = src.globals()
    assert set(g) == {"embed_tokens.weight", "norm.weight"} and all(np.array_equal(g[k], w[k]) for k in g)
    for l in (2, 0, 1, 2):                          # any order: each layer restarts from its own saved state
        t = src.layer(l)
        assert list(t) == [n for n, _ in src.layer_names(l)]
        assert all(t[k].dtype == np.float32 and np.array_equal(t[k], w[k]) for k in t)


def _write_sharded(path, kind, sd, config):
    """a snapshot as transformers saves a sharded one: config.json, model-0000i-of-0000n.safetensors, the index"""
    from safetensors.torch import save_file
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(config, f)
    names = list(sd)
    shards = [names[i::3] for i in range(3)]          # interleaved, so every layer spans several shards
    weight_map = {}
    for i, part in enumerate(shards):
        fn = f"model-{i + 1:05d}-of-00003.safetensors"
        save_file({k: sd[k].contiguous() for k in part}, os.path.join(path, fn))
        weight_map.update({k: fn for k in part})
    with open(os.path.join(path, "model.safetensors.index.json"), "w") as f:
        json.dump({"metadata": {}, "weight_map": weight_map}, f)


@pytest.mark.parametrize("kind", ["llama", "qwen3"])
def test_per_layer_reader_matches_the_whole_snapshot_loader(tmp_path, kind):
    import torch
    H, F, L = 256, 384, 3
    config = {"model_type": kind, "hidden_size": H, "num_attention_heads": 2, "num_key_value_heads": 1,
              "intermediate_size": F, "num_hidden_layers": L, "vocab_size": 300, "max_position_embeddings": 64,
              "rms_norm_eps": 1e-6, "rope_theta": 10000.0, "head_dim": 128, "tie_word_embeddings": False}
    cfg = (LlamaConfig if kind == "llama" else Qwen3Config).from_hf(config)
    from ragmeup_b200.weights import decoder_weight_names
    g = torch.Generator().manual_seed(5)
    sd = {"model." + n: torch.randn(shape, generator=g).to(torch.bfloat16) for n, shape in decoder_weight_names(cfg)}
    sd["lm_head.weight"] = torch.randn(300, H, generator=g).to(torch.bfloat16)   # never read
    _write_sharded(str(tmp_path), kind, sd, config)
    wcfg, w = _load_decoder_snapshot(str(tmp_path))
    src = decoder_layers(str(tmp_path))
    assert src.cfg == wcfg
    got = dict(src.globals())
    for l in range(L):
        t = src.layer(l)
        assert list(t) == [n for n, _ in src.layer_names(l)]
        got.update(t)
    assert set(got) == set(w)
    for k in w:
        assert got[k].dtype == np.float32 and np.array_equal(got[k], w[k]), k


def test_pytorch_model_bin_snapshot_loads_layer_by_layer(tmp_path):
    """a snapshot that ships only pytorch_model.bin still loads: read whole, as _load_decoder_snapshot reads it, then
    handed over one layer at a time"""
    import torch
    H, F, L = 256, 384, 2
    config = {"model_type": "llama", "hidden_size": H, "num_attention_heads": 2, "num_key_value_heads": 1,
              "intermediate_size": F, "num_hidden_layers": L, "vocab_size": 300, "max_position_embeddings": 64,
              "rms_norm_eps": 1e-6, "rope_theta": 10000.0, "head_dim": 128}
    from ragmeup_b200.weights import decoder_weight_names
    cfg = LlamaConfig.from_hf(config)
    g = torch.Generator().manual_seed(6)
    torch.save({"model." + n: torch.randn(shape, generator=g) for n, shape in decoder_weight_names(cfg)},
               os.path.join(str(tmp_path), "pytorch_model.bin"))
    with open(os.path.join(str(tmp_path), "config.json"), "w") as f:
        json.dump(config, f)
    wcfg, w = _load_decoder_snapshot(str(tmp_path))
    src = decoder_layers(str(tmp_path))
    assert src.cfg == wcfg
    got = dict(src.globals())
    for l in range(L):
        got.update(src.layer(l))
    assert set(got) == set(w) and all(np.array_equal(got[k], w[k]) for k in w)


class _Model:
    """a stand-in for a transformers model with CUDA tensors: modules() yields objects with _parameters / _buffers"""

    def __init__(self, tensors, name="some/model"):
        self.name_or_path = name
        self.generation_config = object()
        self._parameters = dict(tensors)
        self._buffers = {}

    def modules(self):
        return [self]


class _T:
    def __init__(self, n, index=0):
        self.n, self.is_cuda, self.dtype = n, True, "float16"
        self.device = type("D", (), {"index": index})()
        self.quant_state = type("Q", (), {"absmax": None})()

    def numel(self):
        return self.n

    def element_size(self):
        return 2


GiB = 1 << 30


def _intact(m):
    return all(not hasattr(t, "data") and t.quant_state is not None for t in m._parameters.values() if t is not None)


def test_release_rule(monkeypatch):
    """the transformers copy goes only when the planned decoder would not fit in the free memory beside it and does
    fit once the copy is freed; otherwise the copy is left as it was"""
    import torch
    from ragmeup_b200 import provenance
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (10 * GiB, 80 * GiB))
    monkeypatch.setattr(torch.cuda, "empty_cache", lambda: None)
    monkeypatch.setattr(torch, "empty", lambda *a, **k: "empty")
    m = _Model({"a": _T(3 * GiB), "b": _T(24), "other_gpu": _T(GiB, index=1), "none": None})  # 6 GiB + 48 B on cuda:0
    assert provenance.release_model_if_needed(m, 5 * GiB, 0) == 0                    # fits: nothing changes
    assert _intact(m)
    with pytest.raises(ValueError, match=r"needs 18253611008 bytes .*=nf4; .* 10737418240 bytes free .* 6442450992 "
                                         r"bytes .* left as it was"):
        provenance.release_model_if_needed(m, 17 * GiB, 0, "nf4")                  # more than freeing could give
    assert _intact(m)
    assert provenance.release_model_if_needed(m, 15 * GiB, 0) == 6 * GiB + 48
    assert m._parameters["a"].data == "empty" and m._parameters["a"].quant_state is None
    assert not hasattr(m._parameters["other_gpu"], "data")                           # another device: kept
    assert m.name_or_path == "some/model" and m.generation_config is not None
    assert provenance.release_model_if_needed("a name", 1 << 50, 0) == 0             # not a model: nothing to free


def test_decoder_refusals_leave_the_model_alone(monkeypatch):
    """provenance._decoder on a transformers model: split weights at the 70B shape are refused before the model is
    touched, and so is an NF4 decoder that would not fit even without the model; neither builds a decoder"""
    import torch
    from ragmeup_b200 import provenance
    made = []

    class FakeTorch:
        class cuda:
            @staticmethod
            def current_device():
                return 0

    monkeypatch.setattr(_lib, "require_cuda", lambda: FakeTorch)
    monkeypatch.setattr(provenance, "_DECODERS", {})
    class Fake:
        def __init__(self, *a, **k):
            made.append(a)

    monkeypatch.setattr(provenance, "DecoderAttention", Fake)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (20 * GiB, 80 * GiB))
    monkeypatch.setattr(torch.cuda, "empty_cache", lambda: None)
    m = _Model({"w": _T(20 * GiB)}, name="synthetic:llama-3.1-70b")               # 40 GiB on cuda:0
    monkeypatch.delenv("RMU_DECODER_WEIGHTS", raising=False)
    with pytest.raises(ValueError, match="RMU_DECODER_WEIGHTS=nf4"):
        provenance._decoder(m)
    assert _intact(m) and not made
    monkeypatch.setenv("RMU_DECODER_WEIGHTS", "nf4")
    small = _Model({"w": _T(GiB)}, name="synthetic:llama-3.1-70b")                # 2 GiB: 22 GiB < 48.96 GB
    with pytest.raises(ValueError, match="left as it was"):
        provenance._decoder(small)
    assert _intact(small) and not made
    monkeypatch.setattr(torch, "empty", lambda *a, **k: "empty")
    provenance._decoder(m)                                                         # 60 GiB once freed: it goes
    assert m._parameters["w"].data == "empty" and made == [("synthetic:llama-3.1-70b",)]
