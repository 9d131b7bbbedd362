"""CPU: attention provenance — the float64 decoder oracle against transformers (Llama and Qwen3 last-layer attention),
the llama3 rope table, LlamaConfig's forms and refusals, the span arithmetic on hand-built attention tensors (oracle and
drop-in alike), and the C refusals of the new entry points."""
import ctypes
import json
import os
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import decoder_attention_ref as da
from ragmeup_b200 import provenance
from ragmeup_b200.weights import (DECODER_PRESETS, PRESETS, LlamaConfig, Qwen3Config, llama_weight_names,
                                  resolve_decoder, rope_table, synthetic_llama_weights, synthetic_qwen3_weights)

# Llama-3.1-8B-Instruct's config.json in its release form [3P-recall] and in transformers 5's form
RELEASE = {"model_type": "llama", "architectures": ["LlamaForCausalLM"], "hidden_size": 4096, "intermediate_size": 14336,
           "num_attention_heads": 32, "num_key_value_heads": 8, "num_hidden_layers": 32, "vocab_size": 128256,
           "max_position_embeddings": 131072, "rms_norm_eps": 1e-5, "hidden_act": "silu", "attention_bias": False,
           "mlp_bias": False, "rope_theta": 500000.0, "tie_word_embeddings": False,
           "rope_scaling": {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                            "original_max_position_embeddings": 8192}}
HF5 = {k: v for k, v in RELEASE.items() if k not in ("rope_scaling", "rope_theta")}
HF5["rope_parameters"] = dict(RELEASE["rope_scaling"], rope_theta=500000.0)


def test_config_forms():
    for d in (RELEASE, HF5):
        cfg = LlamaConfig.from_hf(d)
        assert (cfg.hidden, cfg.heads, cfg.kv_heads, cfg.head_dim, cfg.ffn, cfg.layers) == (4096, 32, 8, 128, 14336, 32)
        assert cfg.rope_theta == 5e5 and cfg.rope_scaling == (8.0, 1.0, 4.0, 8192) and cfg.ln_eps == 1e-5
        assert asdict(cfg) == asdict(DECODER_PRESETS["llama-3.1-8b"]) | {"name": "llama"}
    plain = LlamaConfig.from_hf({k: v for k, v in RELEASE.items() if k != "rope_scaling"})
    assert plain.rope_scaling is None and plain.rope_theta == 5e5
    # Llama-3.2-3B: head_dim 128 (3072 / 24)
    assert LlamaConfig.from_hf(dict(RELEASE, hidden_size=3072, num_attention_heads=24)).head_dim == 128


@pytest.mark.parametrize("field,value,name", [
    ("hidden_act", "gelu", "hidden_act"), ("attention_bias", True, "attention_bias"), ("mlp_bias", True, "mlp_bias"),
    ("rope_scaling", {"rope_type": "yarn", "factor": 4.0}, "rope_type"),
    ("rope_scaling", {"type": "linear", "factor": 2.0}, "rope_type"),
    ("num_attention_heads", 64, "head_dim"),              # Llama-3.2-1B's head_dim 64 (2048 / 32)
    ("model_type", "mistral", "model_type")])
def test_refusals_name_the_field(field, value, name):
    with pytest.raises(ValueError, match=name):
        LlamaConfig.from_hf(dict(RELEASE, **{field: value}))
    if field == "rope_scaling":
        with pytest.raises(ValueError, match=name):
            LlamaConfig.from_hf(dict(HF5, rope_parameters=dict(value, rope_theta=1e4)))


def test_llama3_rope_table_equals_transformers():
    from transformers import LlamaConfig as HFLlamaConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding
    for preset in ("tiny-llama", "llama-3.1-8b"):
        cfg = DECODER_PRESETS[preset]
        f, lo, hi, old = cfg.rope_scaling
        hc = HFLlamaConfig(hidden_size=cfg.hidden, num_attention_heads=cfg.heads, head_dim=cfg.head_dim,
                           max_position_embeddings=cfg.max_pos, rope_theta=cfg.rope_theta,
                           rope_scaling={"rope_type": "llama3", "factor": f, "low_freq_factor": lo, "high_freq_factor": hi,
                                         "original_max_position_embeddings": old})
        rot = LlamaRotaryEmbedding(hc)
        rows = min(cfg.max_pos, 16384)
        cos, sin = rot(torch.zeros(1, dtype=torch.float32), torch.arange(rows)[None])
        mine = rope_table(cfg.rope_theta, cfg.head_dim, rows, cfg.rope_scaling)
        assert np.array_equal(mine[0], cos[0, :, :cfg.head_dim // 2].numpy()), preset
        assert np.array_equal(mine[1], sin[0, :, :cfg.head_dim // 2].numpy()), preset
        plain = rope_table(cfg.rope_theta, cfg.head_dim, 64)
        assert not np.array_equal(mine[0][:64], plain[0]), "the scaling changes some frequencies"


def _hf_float64(monkeypatch, module, norm_cls):
    """transformers' eager softmax and RMSNorm upcast run in float32 whatever the model's dtype: keep them in float64"""
    sm = torch.nn.functional.softmax
    monkeypatch.setattr(torch.nn.functional, "softmax", lambda x, dim=-1, dtype=None: sm(x, dim=dim))

    def rms64(self, x):
        return self.weight * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.variance_epsilon))
    monkeypatch.setattr(getattr(module, norm_cls), "forward", rms64)


def _hf_state(w):
    return {"model." + k: torch.from_numpy(v).double() for k, v in w.items()}


@pytest.mark.parametrize("family", ["llama", "qwen3"])
def test_oracle_last_attention_matches_transformers_float64(monkeypatch, family):
    """the float64 oracle's last-layer probabilities against transformers' eager ``attentions[-1]`` in float64: GQA,
    llama3 scaling and no q / k norm (Llama), q / k norm (Qwen3); |delta| <= 1e-12"""
    import transformers
    if family == "llama":
        from transformers.models.llama import modeling_llama as m
        cfg = LlamaConfig(**asdict(DECODER_PRESETS["tiny-llama"]))
        w = synthetic_llama_weights(cfg, seed=3)
        f, lo, hi, old = cfg.rope_scaling
        hc = transformers.LlamaConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, intermediate_size=cfg.ffn,
                                      num_hidden_layers=cfg.layers, num_attention_heads=cfg.heads,
                                      num_key_value_heads=cfg.kv_heads, head_dim=cfg.head_dim,
                                      max_position_embeddings=cfg.max_pos, rms_norm_eps=cfg.ln_eps,
                                      rope_theta=cfg.rope_theta, tie_word_embeddings=False, attn_implementation="eager",
                                      rope_scaling={"rope_type": "llama3", "factor": f, "low_freq_factor": lo,
                                                    "high_freq_factor": hi, "original_max_position_embeddings": old})
        model = transformers.LlamaForCausalLM(hc)
        _hf_float64(monkeypatch, m, "LlamaRMSNorm")
    else:
        from transformers.models.qwen3 import modeling_qwen3 as m
        cfg = Qwen3Config(**asdict(PRESETS["tiny-qwen3"][0]))
        w = synthetic_qwen3_weights(cfg, seed=3)
        hc = transformers.Qwen3Config(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, intermediate_size=cfg.ffn,
                                      num_hidden_layers=cfg.layers, num_attention_heads=cfg.heads,
                                      num_key_value_heads=cfg.kv_heads, head_dim=cfg.head_dim,
                                      max_position_embeddings=cfg.max_pos, rms_norm_eps=cfg.ln_eps,
                                      rope_theta=cfg.rope_theta, tie_word_embeddings=False, attn_implementation="eager")
        model = transformers.Qwen3ForCausalLM(hc)
        _hf_float64(monkeypatch, m, "Qwen3RMSNorm")
    model = model.double().eval()
    missing, unexpected = model.load_state_dict(_hf_state(w), strict=False)
    assert not unexpected and all(k == "lm_head.weight" for k in missing)
    ids = np.random.default_rng(5).integers(0, cfg.vocab_size, 150).tolist()
    with torch.no_grad():
        want = model(input_ids=torch.tensor([ids]), output_attentions=True).attentions[-1][0]
    got = da.last_attention(w, cfg, ids, qk_norm=family == "qwen3")
    assert got.shape == want.shape and float((got - want).abs().max()) <= 1e-12


# ---------------------------------------------------------------------------------------------------- span arithmetic
class _FromTensor(provenance.DecoderAttention):
    """the drop-in's arithmetic over a given attention tensor: span_mass sums A over the spans as the GPU would"""
    def __init__(self, A):
        self.A = A
        self.cfg = LlamaConfig(heads=A.shape[0], name="hand-built")

    def span_mass(self, ids, spans):
        return np.array([[self.A[:, a0:a1, b0:b1].sum() for b0, b1 in spans] for a0, a1 in spans])


class _Tok:
    def encode(self, text, add_special_tokens=True):
        assert add_special_tokens is False
        return [int(t) for t in text.split()]


def _attn(T, heads=2, seed=0):
    x = np.random.default_rng(seed).standard_normal((heads, T, T))
    x = np.where(np.tril(np.ones((T, T), bool)), x, -np.inf)
    e = np.exp(x - x.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def _both(A, thread, query, context, answer):
    tok = _Tok()
    want = da.attention_scores(A, tok.encode(thread, False), tok.encode(query, False), tok.encode(answer, False),
                               [tok.encode(c, False) for c in context],
                               include_query=os.getenv("attribute_include_query") != "False")
    got = provenance.compute_attention(_FromTensor(A), tok, thread, query, context, answer)
    assert all(isinstance(g, np.float64) for g in got)
    np.testing.assert_allclose(got, want, rtol=1e-12, equal_nan=True)
    return got


def _by_hand(A, q, a, docs, include_query=True):
    def mean(r, c):
        blk = A[:, r[0]:r[1], c[0]:c[1]]
        return blk.mean() if blk.size else np.nan
    total = [v for v in (mean(q, q), mean(q, a), mean(a, a), mean(a, q)) if v > 0]
    out = []
    for d in docs:
        vals = [mean(a, d), mean(d, a)] + ([mean(q, d), mean(d, q)] if include_query else [])
        kept = [v for v in vals if v > 0]
        total += kept
        out.append(np.mean(kept) if kept else np.nan)
    return [s / np.mean(total) for s in out]


THREAD = "90 91 10 11 12 92 20 21 22 23 93 30 31 32 94 40 41 42 43 95 50 51 52 96"


@pytest.mark.parametrize("setting", [None, "True", "False"])
def test_span_arithmetic_by_hand(monkeypatch, setting):
    if setting is None:
        monkeypatch.delenv("attribute_include_query", raising=False)
    else:
        monkeypatch.setenv("attribute_include_query", setting)
    A = _attn(24)
    got = _both(A, THREAD, "40 41 42 43", ["10 11 12", "20 21 22 23", "30 31 32"], "50 51 52")
    # the slices leave each part's last token out: query [15:18], answer [20:22], documents [2:4], [6:9], [11:13]
    want = _by_hand(A, (15, 18), (20, 22), [(2, 4), (6, 9), (11, 13)], include_query=setting != "False")
    np.testing.assert_allclose(got, want, rtol=1e-12)


def test_one_token_part_and_empty_answer(monkeypatch):
    monkeypatch.delenv("attribute_include_query", raising=False)
    A = _attn(24, seed=1)
    # a one-token document is an empty slice: its blocks are NaN, so nothing is kept and its score is NaN
    got = _both(A, THREAD, "40 41 42 43", ["10 11 12", "30"], "50 51 52")
    assert np.isnan(got[1]) and np.isfinite(got[0])
    # an empty answer is found at 0 and slices [0:-1]: every row but the last
    got = _both(A, THREAD, "40 41 42 43", ["10 11 12", "20 21 22 23"], "")
    np.testing.assert_allclose(got, _by_hand(A, (15, 18), (0, 23), [(2, 4), (6, 9)]), rtol=1e-12)


def test_document_without_positive_block_scores_nan(monkeypatch):
    monkeypatch.setenv("attribute_include_query", "False")
    A = _attn(24, seed=2)
    A[:, :, 2:4] = 0.0          # no attention reaches document 0, and its rows look at nothing of the answer
    A[:, 2:4, :] = 0.0
    got = _both(A, THREAD, "40 41 42 43", ["10 11 12", "20 21 22 23"], "50 51 52")
    assert np.isnan(got[0]) and np.isfinite(got[1])


def test_repeated_document_takes_the_first_occurrence(monkeypatch):
    monkeypatch.delenv("attribute_include_query", raising=False)
    A = _attn(30, seed=3)
    thread = THREAD + " 20 21 22 23 97"
    got = _both(A, thread, "40 41 42 43", ["20 21 22 23", "20 21 22 23"], "50 51 52")
    assert got[0] == got[1]
    np.testing.assert_allclose(got, _by_hand(A, (15, 18), (20, 22), [(6, 9), (6, 9)]), rtol=1e-12)


def test_missing_part_raises():
    A = _attn(24)
    for q, c, a in (("77", ["10 11 12"], "50 51"), ("40 41", ["10 12"], "50 51"), ("40 41", ["10 11"], "51 50")):
        with pytest.raises(ValueError, match="Sublist not found"):
            provenance.compute_attention(_FromTensor(A), _Tok(), THREAD, q, c, a)
        with pytest.raises(ValueError, match="Sublist not found"):
            da.attention_scores(A, _Tok().encode(THREAD, False), _Tok().encode(q, False), _Tok().encode(a, False),
                                [_Tok().encode(x, False) for x in c])


# ---------------------------------------------------------------------------------------------------- presets, loader
def test_decoder_presets_and_snapshots(tmp_path):
    cfg, w = resolve_decoder("synthetic:tiny-llama")
    assert isinstance(cfg, LlamaConfig) and cfg.head_dim == 128 and cfg.heads == 2 * cfg.kv_heads and cfg.layers in (2, 3)
    assert [n for n, _ in llama_weight_names(cfg)] == list(w) and not any("q_norm" in n for n in w)
    qcfg, qw = resolve_decoder("synthetic:tiny-qwen3")
    assert isinstance(qcfg, Qwen3Config) and "head" not in qw and "layers.0.self_attn.q_norm.weight" in qw
    # a sharded bf16 snapshot under model. with an lm_head: read as fp32, lm_head never read
    from safetensors.torch import save_file
    import torch as T
    d = tmp_path / "llama"
    d.mkdir()
    (d / "config.json").write_text(json.dumps(dict(RELEASE, hidden_size=256, num_attention_heads=2,
                                                   num_key_value_heads=1, num_hidden_layers=cfg.layers,
                                                   intermediate_size=384, vocab_size=1000)))
    small = LlamaConfig.from_hf(json.loads((d / "config.json").read_text()))
    sw = synthetic_llama_weights(small, seed=1)
    bf = {("model." + k): T.from_numpy(v).to(T.bfloat16) for k, v in sw.items()}
    bf["lm_head.weight"] = T.zeros(3, 3, dtype=T.bfloat16)
    names = sorted(bf)
    half = len(names) // 2
    save_file({k: bf[k] for k in names[:half]}, str(d / "model-00001-of-00002.safetensors"))
    save_file({k: bf[k] for k in names[half:]}, str(d / "model-00002-of-00002.safetensors"))
    (d / "model.safetensors.index.json").write_text(json.dumps({"weight_map": {
        k: ("model-00001-of-00002.safetensors" if i < half else "model-00002-of-00002.safetensors")
        for i, k in enumerate(names)}}))
    c2, w2 = resolve_decoder(str(d))
    assert isinstance(c2, LlamaConfig) and set(w2) == set(sw)
    for k, v in sw.items():
        assert w2[k].dtype == np.float32 and np.array_equal(w2[k], T.from_numpy(v).to(T.bfloat16).float().numpy()), k


def test_other_products_keep_refusing_llama(tmp_path):
    from ragmeup_b200.weights import MODEL_TYPES, load_hf_snapshot, resolve_model
    assert "llama" not in MODEL_TYPES
    (tmp_path / "config.json").write_text(json.dumps(RELEASE))
    with pytest.raises(ValueError, match="model_type 'llama' is not supported"):
        load_hf_snapshot(str(tmp_path), with_head=False)
    with pytest.raises(ValueError, match="unknown synthetic preset"):
        resolve_model("synthetic:tiny-llama", with_head=False)


def test_compute_attention_fails_loudly_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from ragmeup_b200 import _lib
    with pytest.raises(_lib.RmuError):
        provenance.compute_attention("synthetic:tiny-llama", _Tok(), "1 2 3", "1", [], "2")
    with pytest.raises(_lib.RmuError):
        provenance.DecoderAttention("synthetic:tiny-llama")


# ---------------------------------------------------------------------------------------------------- C refusals
def test_c_refusals_before_any_cuda_call():
    """rmu_encoder_create_llama, rmu_decoder_attention_spans and rmu_debug_attention_spans refuse bad arguments before
    any CUDA call (pointers are stand-ins, never dereferenced; the machine may have no GPU)"""
    from ragmeup_b200 import _lib
    l = _lib.lib()
    ERR_ARG, UNSUP = -1, -3
    p = 1 << 20
    cfg = LlamaConfig(**asdict(DECODER_PRESETS["tiny-llama"]))
    w = synthetic_llama_weights(cfg, seed=0)
    cos, sin = cfg.rope_tables()

    def create(cfg=cfg, w=w, head_form=0, extra=0, drop=0, **kw):
        arrs = [np.ascontiguousarray(w[n]) for n, _ in llama_weight_names(cfg)] + [cos, sin]
        arrs = arrs[:len(arrs) - drop] + [cos] * extra
        ptrs = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        cc = _lib.bert_config_c(cfg)
        qx = _lib.Qwen3ExtC(kw.get("kv", cfg.kv_heads), kw.get("hd", 128), cfg.max_pos, 64, head_form, -1)
        h = ctypes.c_void_p()
        rc = l.rmu_encoder_create_llama(ctypes.byref(cc), ctypes.byref(qx), ptrs, len(arrs), ctypes.byref(h))
        if rc == 0:
            l.rmu_encoder_destroy(h)
        return rc

    assert create(head_form=1) == ERR_ARG and b"RMU_QWEN3_HEAD_NONE" in l.rmu_last_error()
    assert create(extra=1) == ERR_ARG and create(drop=1) == ERR_ARG and b"weight tensors" in l.rmu_last_error()
    assert create(hd=64) == UNSUP and b"head_dim" in l.rmu_last_error()
    assert create(kv=3) == UNSUP
    for field, value in (("hidden", 320), ("hidden", 4224), ("ffn", 100)):
        c = LlamaConfig(**{**asdict(cfg), field: value})
        assert create(cfg=c) == UNSUP, (field, value)
    for name in ("layers.1.self_attn.k_proj.weight", "layers.0.mlp.down_proj.weight", "layers.2.self_attn.o_proj.weight"):
        bad = dict(w)
        bad[name] = w[name].copy()
        bad[name].reshape(-1)[5] = 7e4
        assert create(w=bad) == UNSUP and b"65520" in l.rmu_last_error(), name
    assert create() in (0, -2)                           # accepted: without a device the next step fails
    assert l.rmu_encoder_create_llama(None, None, None, 0, None) == ERR_ARG

    fake = ctypes.c_void_p(p)
    for T, n, ids, spans, out in ((0, 2, p, p, p), (-1, 2, p, p, p), (5, 0, p, p, p), (5, 2, None, p, p),
                                  (5, 2, p, None, p), (5, 2, p, p, None)):
        assert l.rmu_decoder_attention_spans(fake, ids, T, spans, n, out, None) == ERR_ARG
    assert l.rmu_decoder_attention_spans(None, p, 5, p, 2, p, None) == ERR_ARG
    assert b"rmu_decoder_attention_spans" in l.rmu_last_error()

    def dbg(T=17, heads=8, kv=2, n=3, **kw):
        a = dict(hi=p, lo=p, spans=p, out=p)
        a.update(kw)
        return l.rmu_debug_attention_spans(a["hi"], a["lo"], T, heads, kv, a["spans"], n, a["out"], None)

    assert dbg(heads=6, kv=4) == UNSUP and b"rmu_debug_attention_spans" in l.rmu_last_error()
    for kw in ({"T": 0}, {"heads": 0}, {"kv": 0}, {"n": 0}, {"n": -1}, {"hi": None}, {"lo": None}, {"spans": None},
               {"out": None}):
        assert dbg(**kw) == ERR_ARG, kw


# ---------------------------------------------------------------------------------------------------- goldens
def _golden_module():
    import importlib.util
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden_llama.py")
    spec = importlib.util.spec_from_file_location("make_golden_llama", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_golden_script_reproduces_the_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "llama.npz"))
    with torch.no_grad():
        new = _golden_module().compute()
    assert set(new) == set(g.files)
    for k in g.files:
        assert new[k].dtype == g[k].dtype and np.array_equal(new[k], g[k], equal_nan=k.startswith("scores")), k


@pytest.mark.parametrize("setting,key", [("True", "scores_q"), ("False", "scores_noq")])
def test_golden_scores_follow_from_the_golden_mass(monkeypatch, golden_dir, setting, key):
    """the drop-in's arithmetic on the fixture's span masses gives the fixture's scores (the oracle's, from the full
    attention tensor)"""
    monkeypatch.setenv("attribute_include_query", setting)
    g = np.load(os.path.join(golden_dir, "llama.npz"))
    mod = _golden_module()

    class FromMass(provenance.DecoderAttention):
        def __init__(self):
            self.cfg = LlamaConfig(**asdict(DECODER_PRESETS["tiny-llama"]))

        def span_mass(self, ids, spans):
            assert list(ids) == g["ids"].tolist() and [tuple(s) for s in spans] == [tuple(s) for s in g["spans"].tolist()]
            return g["mass"]

    text, query, docs, answer = mod.thread()
    got = provenance.compute_attention(FromMass(), mod.tokenizer(), text, query, docs, answer)
    np.testing.assert_allclose(got, g[key], rtol=1e-12, equal_nan=True)
    assert np.isnan(got[-1])                                # the one-token document


def test_decoder_oracle_is_the_qwen3_oracle_with_qk_norm():
    """decoder_attention_ref's forward with qk_norm=True is qwen3_ref's, bit for bit, so the two stay in step"""
    from oracle import qwen3_ref
    cfg = Qwen3Config(**asdict(PRESETS["tiny-qwen3"][0]))
    w = qwen3_ref.weights(synthetic_qwen3_weights(cfg, seed=4, scale=2.0))
    ids = np.random.default_rng(6).integers(0, cfg.vocab_size, 90).tolist()
    with torch.no_grad():
        assert torch.equal(da.hidden(w, cfg, ids, qk_norm=True), qwen3_ref.hidden(w, cfg, ids))
