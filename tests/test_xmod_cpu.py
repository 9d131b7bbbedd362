"""CPU: X-MOD checkpoints (ColBERT-XM's backbone).  Config refusals, language selection, reading one language's
adapters only, the oracle against transformers' XmodModel / XmodForSequenceClassification (live, and the golden minted
by tests/golden/make_golden_xmod.py), ColBERT tokenisation on the synthetic SentencePiece Unigram vocabulary, the C
config's new field and rmu_encoder_create's adapter refusals (which come before any CUDA call)."""
import ctypes
import json
import os
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import bert_ref, xmod_ref
from ragmeup_b200 import weights as W
from ragmeup_b200.colbert import ColBERTTokenizer
from ragmeup_b200.tokenizer import load_tokenizer
from ragmeup_b200.weights import PRESETS, XmodConfig, synthetic_bert_weights, weight_names

LANGS = ("en_XX", "de_DE", "fr_XX")


def _cfg(preset="tiny-xmod", **kw):
    return XmodConfig(**{**asdict(PRESETS[preset][0]), **kw})


def _hf_conf(cfg, **kw):
    d = {"model_type": "xmod", "vocab_size": cfg.vocab_size, "hidden_size": cfg.hidden,
         "num_hidden_layers": cfg.layers, "num_attention_heads": cfg.heads, "intermediate_size": cfg.ffn,
         "max_position_embeddings": cfg.max_pos, "type_vocab_size": 1, "layer_norm_eps": cfg.ln_eps, "pad_token_id": 1,
         "adapter_reduction_factor": cfg.hidden // cfg.adapter_dim, "languages": list(cfg.languages),
         "default_language": cfg.languages[0], "pre_norm": False, "adapter_layer_norm": False,
         "adapter_reuse_layer_norm": True, "ln_before_adapter": True}
    d.update(kw)
    return d


@pytest.fixture(autouse=True)
def _no_language_env(monkeypatch):
    monkeypatch.delenv(W.XMOD_LANGUAGE_ENV, raising=False)


# ----------------------------------------------------------------------------------------------- config refusals
@pytest.mark.parametrize("patch,match", [
    ({"pre_norm": True}, "pre_norm"),
    ({"adapter_layer_norm": True}, "adapter_layer_norm"),
    ({"adapter_reuse_layer_norm": False}, "adapter_reuse_layer_norm"),
    ({"ln_before_adapter": False}, "ln_before_adapter"),
    ({"adapter_reduction_factor": 3}, "adapter_reduction_factor"),
    ({"pad_token_id": 0}, "pad_token_id"),
    ({"position_embedding_type": "relative_key"}, "absolute"),
    ({"hidden_act": "relu"}, "erf-GELU"),
])
def test_config_refusals(tmp_path, patch, match):
    cfg = _cfg()
    with pytest.raises(ValueError, match=match):
        XmodConfig.from_hf(_hf_conf(cfg, **patch))
    # from a snapshot, before any tensor is read (there is none)
    os.makedirs(tmp_path / "m")
    with open(tmp_path / "m" / "config.json", "w") as f:
        json.dump(_hf_conf(cfg, **patch), f)
    with pytest.raises(ValueError, match=match):
        W.resolve_model(str(tmp_path / "m"), with_head=False)


def test_config_fields():
    c = XmodConfig.from_hf(_hf_conf(_cfg()))
    assert (c.adapter_dim, c.languages, c.language, c.position_mode, c.type_vocab) == (128, LANGS, "en_XX", 1, 1)
    # transformers' defaults where config.json leaves the flags out
    d = _hf_conf(_cfg())
    for k in ("pre_norm", "adapter_layer_norm", "adapter_reuse_layer_norm", "ln_before_adapter", "adapter_reduction_factor"):
        d.pop(k)
    assert XmodConfig.from_hf(d).adapter_dim == 128
    assert W.BertConfig().adapter_dim == 0 and W.XLMRConfig().adapter_dim == 0
    assert "adapter_dim" not in asdict(W.BertConfig()) and "adapter_dim" not in asdict(W.XLMRConfig())


# ------------------------------------------------------------------------------------------- language selection
def test_language_precedence(monkeypatch):
    d = _hf_conf(_cfg(), default_language="de_DE")
    assert XmodConfig.from_hf(d).language == "de_DE"
    monkeypatch.setenv(W.XMOD_LANGUAGE_ENV, "fr_XX")                  # the environment overrides the default
    assert XmodConfig.from_hf(d).language == "fr_XX"
    assert XmodConfig.from_hf({**d, "default_language": None}).language == "fr_XX"
    monkeypatch.setenv(W.XMOD_LANGUAGE_ENV, "xx_YY")
    with pytest.raises(ValueError, match="language 'xx_YY': it is not one of"):
        XmodConfig.from_hf(d)
    monkeypatch.delenv(W.XMOD_LANGUAGE_ENV)
    with pytest.raises(ValueError, match=r"model_type 'xmod' is not supported without an input language.*\['en_XX', 'de_DE', 'fr_XX'\]"):
        XmodConfig.from_hf({**d, "default_language": None})
    with pytest.raises(ValueError, match="is not one of"):
        XmodConfig.from_hf({**d, "default_language": "it_IT"})
    # synthetic presets: the preset's language is the default, the environment overrides it
    assert W.resolve_model("synthetic:tiny-xmod", with_head=False)[0].language == "en_XX"
    monkeypatch.setenv(W.XMOD_LANGUAGE_ENV, "de_DE")
    assert W.resolve_model("synthetic:tiny-xmod", with_head=False)[0].language == "de_DE"
    assert W.resolve_colbert("synthetic:colbert-xm")[0].language == "de_DE"


# --------------------------------------------------------------------------------------------------- snapshots
def _hf_model(cfg, head, default_language="en_XX"):
    from transformers import XmodConfig as HC, XmodForSequenceClassification, XmodModel
    d = _hf_conf(cfg, default_language=default_language)
    hc = HC(**{k: v for k, v in d.items() if k != "model_type"}, hidden_dropout_prob=0.0,
            attention_probs_dropout_prob=0.0, attn_implementation="eager", num_labels=1)
    return (XmodForSequenceClassification(hc) if head else XmodModel(hc, add_pooling_layer=False)).eval()


def _canonical(sd):
    out = {}
    for k, v in sd.items():
        k = k.replace("roberta.", "", 1)
        if k.startswith("classifier.dense."):
            k = "pooler.dense." + k[len("classifier.dense."):]
        elif k.startswith("classifier.out_proj."):
            k = "classifier." + k[len("classifier.out_proj."):]
        out[k] = v.detach().numpy()
    return out


@pytest.mark.parametrize("head", [False, True])
def test_only_the_selected_language_is_read(tmp_path, monkeypatch, head):
    import safetensors
    torch.manual_seed(1)
    m = _hf_model(_cfg(), head)
    path = str(tmp_path / "xmod")
    m.save_pretrained(path)
    want = _canonical(m.state_dict())
    read = []
    real = safetensors.safe_open

    class Spy:
        def __init__(self, *a, **k):
            self.f = real(*a, **k)

        def __enter__(self):
            self.f.__enter__()
            return self

        def __exit__(self, *a):
            return self.f.__exit__(*a)

        def keys(self):
            return self.f.keys()

        def get_tensor(self, k):
            read.append(k)
            return self.f.get_tensor(k)

    monkeypatch.setattr(safetensors, "safe_open", Spy)
    monkeypatch.setenv(W.XMOD_LANGUAGE_ENV, "de_DE")
    cfg, w, *_ = W.resolve_model(path, with_head=head)
    adapters = [k for k in read if ".adapter_modules." in k]
    assert adapters and all(".adapter_modules.de_DE." in k for k in adapters)
    assert len(adapters) == 4 * cfg.layers
    assert not any(".adapter_modules." in k and ".de_DE." not in k for k in w)
    for name, shape in weight_names(cfg, head):
        assert w[name].shape == shape and np.array_equal(w[name], want[name]), name
    assert weight_names(cfg, head)[-1][0] == f"encoder.layer.{cfg.layers - 1}.output.adapter_modules.de_DE.dense2.bias"


def test_oracle_matches_transformers_for_two_languages():
    """XmodModel and XmodForSequenceClassification with random init against the fp32 oracle, one language at a time;
    the two languages' outputs differ, so the adapter ran"""
    from transformers import XmodForSequenceClassification
    cfg = _cfg()
    torch.manual_seed(3)
    m = _hf_model(cfg, True)
    assert isinstance(m, XmodForSequenceClassification)
    with torch.no_grad():                 # trained-like adapters: the random init's are small
        for n, p in m.named_parameters():
            if ".adapter_modules." in n:
                p.mul_(4.0)
    w = _canonical(m.state_dict())
    ids = torch.tensor([[0, 17, 1, 99, 2, 5, 6, 2], [0, 33, 44, 2, 1, 1, 1, 1]])
    mask = torch.tensor([[1] * 8, [1] * 4 + [0] * 4])
    outs = {}
    for lang in ("de_DE", "fr_XX"):
        ocfg = xmod_ref.XmodCfg(**{**asdict(cfg), "language": lang})
        with torch.no_grad():
            r = m(input_ids=ids, attention_mask=mask, lang_ids=torch.full((2,), LANGS.index(lang)), output_hidden_states=True)
            h = xmod_ref.xmod_encoder_forward(w, ocfg, ids, mask)
            lg = xmod_ref.classifier_head(w, h)
        valid = mask.bool()
        assert float((h - r.hidden_states[-1])[valid].abs().max()) < 4e-6
        assert float((lg - r.logits).abs().max()) < 4e-6
        outs[lang] = h[valid]
    assert float((outs["de_DE"] - outs["fr_XX"]).abs().max()) > 1e-2
    # without lang_ids transformers takes default_language, the language the oracle takes from the config
    with torch.no_grad():
        r = m(input_ids=ids, attention_mask=mask)
        h = xmod_ref.xmod_encoder_forward(w, xmod_ref.XmodCfg(**asdict(cfg)), ids, mask)
    assert float((xmod_ref.classifier_head(w, h) - r.logits).abs().max()) < 4e-6


GOLDEN = [("tiny-xmod", 0, 1.0), ("tiny-xmod", 2, 4.0)]


@pytest.mark.parametrize("preset,seed,scale", GOLDEN)
def test_oracle_matches_golden(golden_dir, preset, seed, scale):
    """the fp32 forward and the float64 ragged stack against transformers' outputs for the third language (neither
    the first nor the default), at the bar of test_xlmr_cpu.py"""
    g = np.load(f"{golden_dir}/xmod.npz")
    key = f"xmod_{preset}_{seed}_{scale}"
    cfg = _cfg(preset, languages=LANGS, language="fr_XX")
    w = synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale)
    ids = torch.from_numpy(g[key + "_ids"].astype(np.int64))
    mask = torch.from_numpy(g[key + "_mask"].astype(np.int64))
    lens = mask.sum(1).tolist()
    tol = 4e-6 if scale == 1.0 else 2e-5
    with torch.no_grad():
        h = xmod_ref.xmod_encoder_forward(w, xmod_ref.XmodCfg(**asdict(cfg)), ids, mask)
        other = xmod_ref.xmod_encoder_forward(w, xmod_ref.XmodCfg(**asdict(cfg)), ids, mask, language="de_DE")
    assert np.abs(bert_ref.l2_normalize(bert_ref.pool(h, mask, "mean")).numpy() - g[key + "_mean"]).max() < tol
    assert np.abs(h[:, 0].numpy() - g[key + "_h_first"]).max() < 50 * tol
    assert np.abs(other[:, 0].numpy() - g[key + "_h_first"]).max() > 1e3 * tol       # the language matters
    want = g[key + "_logits"]
    assert np.abs(xmod_ref.classifier_head(w, h).numpy() - want).max() < 50 * tol * max(1.0, float(np.abs(want).max()))
    flat = np.concatenate([g[key + "_ids"][b, :n] for b, n in enumerate(lens)])
    cu = np.r_[0, np.cumsum(lens)]
    ref = xmod_ref.xmod_stack_ref(w, cfg, flat, cu)
    assert float((ref["cls_norm"] - torch.from_numpy(g[key + "_cls"]).double()).abs().max()) < tol
    assert float((ref["hidden"][cu[1:] - 1] - torch.from_numpy(g[key + "_h_last"]).double()).abs().max()) < 50 * tol
    assert float((ref["logits"] - torch.from_numpy(want).double()).abs().max()) < 50 * tol * max(1.0, float(np.abs(want).max()))


# ------------------------------------------------------------------------------------ ColBERT on a Unigram vocabulary
TOK = load_tokenizer(None, 2000, xlmr=True)
V = TOK.get_vocab()
BOS, EOS, PAD, UNK, MASK = 0, 2, 1, 3, V["<mask>"]


def _pieces(n, seed=0):
    """n word-initial pieces that tokenise to themselves"""
    cand = sorted(p for p in V if p.startswith("▁") and len(p) > 3 and p[1:].isalpha())
    rng = np.random.default_rng(seed)
    return [cand[int(i)] for i in rng.choice(len(cand), n, replace=False)]


def test_colbert_tokens_by_hand():
    spec = W.ColBERTSpec(query_maxlen=8, doc_maxlen=8)
    t = ColBERTTokenizer(TOK, spec)
    assert (t.cls, t.sep, t.mask, t.pad, t.q_marker, t.d_marker) == (BOS, EOS, MASK, PAD, UNK, UNK)   # markers: <unk>
    a, b, c = _pieces(3)
    ia, ib, ic = V[a], V[b], V[c]
    text = lambda *p: " ".join(x[1:] for x in p)  # noqa: E731
    ids, cu, nk = t.queries([text(a, b), "", text(a, b, c, a, b, c, a), "<pad> " + text(a)])
    S = V["▁"]                            # Metaspace: the space of ". " before nothing, or before a special, is "▁"
    assert ids.reshape(4, 8).tolist() == [[BOS, UNK, ia, ib, EOS, MASK, MASK, MASK],
                                          [BOS, UNK, S, EOS, MASK, MASK, MASK, MASK],
                                          [BOS, UNK, ia, ib, ic, ia, ib, EOS],
                                          [BOS, UNK, S, MASK, ia, EOS, MASK, MASK]]         # a literal <pad> -> <mask>
    assert nk.tolist() == [5, 4, 8, 6]
    # documents: the keep-mask drops the pad id and the skiplist, "first id of each punctuation character" as this
    # tokenizer yields it: "▁" for a character the vocabulary lacks, "▁." for "." (colbert-ai's rule, kept as it is)
    assert S in t.skiplist and V["▁."] in t.skiplist and BOS not in t.skiplist and EOS not in t.skiplist
    assert t.skiplist.tolist() == sorted({TOK.encode(ch, add_special_tokens=False).ids[0]
                                          for ch in "!\"#$%&'()*+,-./:;<=>?@[\\]^_`{|}~"})
    ids, cu, keep = t.docs([text(a) + " . " + text(b) + " <pad>", ""])
    assert ids.tolist() == [BOS, UNK, ia, V["▁."], ib, S, PAD, EOS, BOS, UNK, S, EOS]
    assert keep.tolist() == [1, 1, 1, 0, 1, 0, 0, 1, 1, 1, 0, 1]
    # markers the vocabulary has are used as they are
    t2 = ColBERTTokenizer(TOK, W.ColBERTSpec(query_maxlen=8, doc_maxlen=8, query_token=a, doc_token=b))
    assert (t2.q_marker, t2.d_marker) == (ia, ib)


def test_colbert_tokenisation_matches_oracle():
    rng = np.random.default_rng(5)
    words = [p[1:] for p in _pieces(200, 6)] + list(".,;:!?()-'\"#")
    texts = ["", "x", "<mask> a", "<pad>", "<s> </s>"] + [" ".join(rng.choice(words, int(rng.integers(1, 80))))
                                                           for _ in range(40)]
    for spec in (W.ColBERTSpec(), W.ColBERTSpec(query_maxlen=8, doc_maxlen=12)):
        t = ColBERTTokenizer(TOK, spec)
        ids, cu, nk = t.queries(texts)
        rid, ram = xmod_ref.tokenize_queries(TOK, spec, texts)
        assert ids.reshape(len(texts), -1).tolist() == rid.tolist()
        assert nk.tolist() == ram.sum(1).tolist()
        ids, cu, keep = t.docs(texts)
        rid, ram, rkeep = xmod_ref.tokenize_docs(TOK, spec, texts)
        for b in range(len(texts)):
            n = int(ram[b].sum())
            assert ids[cu[b]:cu[b + 1]].tolist() == rid[b, :n].tolist()
            assert keep[cu[b]:cu[b + 1]].astype(bool).tolist() == rkeep[b, :n].tolist()


def _colbert_snapshot(path, cfg, w, lin, kind="xmod", prefix="roberta."):
    from safetensors.numpy import save_file
    os.makedirs(path, exist_ok=True)
    conf = _hf_conf(cfg, model_type=kind, architectures=["HF_ColBERT"]) if kind == "xmod" else \
        {"model_type": kind, "architectures": ["HF_ColBERT"], "vocab_size": cfg.vocab_size, "hidden_size": cfg.hidden,
         "num_hidden_layers": cfg.layers, "num_attention_heads": cfg.heads, "intermediate_size": cfg.ffn,
         "max_position_embeddings": cfg.max_pos, "type_vocab_size": 1, "pad_token_id": 1}
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(conf, f)
    save_file({**{prefix + k: v for k, v in w.items()}, "linear.weight": lin}, os.path.join(path, "model.safetensors"))
    TOK.save(os.path.join(path, "tokenizer.json"))
    return str(path)


def test_colbert_model_types(tmp_path, monkeypatch):
    """ColBERT runs on bert, xlm-roberta, roberta and xmod encoders, not on MPNet; colbert-xm's language follows the
    rules of any X-MOD snapshot, and an unknown one is refused before anything is read"""
    with pytest.raises(ValueError, match="multiple of 128"):
        W.colbert_spec(None, 200)
    assert W.colbert_spec(None, 96).dim == 96 and W.colbert_spec(None, 256).dim == 256
    cfg, w, lin, _ = W.synthetic_colbert("tiny-colbert-xm", 1)
    p = _colbert_snapshot(tmp_path / "colbert-xm", cfg, w, lin)
    got = W.resolve_colbert(p)
    assert got is not None and isinstance(got[0], XmodConfig) and got[0].language == "en_XX" and got[4] == p
    for name, _ in weight_names(got[0], False):
        assert np.array_equal(got[1][name], w[name]), name
    assert (got[3].query_token, got[3].doc_token, got[3].query_maxlen, got[3].doc_maxlen) == ("[unused0]", "[unused1]",
                                                                                          32, 220)
    monkeypatch.setenv(W.XMOD_LANGUAGE_ENV, "fr_XX")
    got = W.resolve_colbert(p)
    assert got[0].language == "fr_XX" and np.array_equal(got[1][weight_names(got[0], False)[-1][0]],
                                                         w[weight_names(got[0], False)[-1][0]])
    # a language the checkpoint lacks, or none at all: not taken as ColBERT, and refused by resolve_model (the path
    # HuggingFaceCrossEncoder takes next) before a tensor is read
    monkeypatch.setenv(W.XMOD_LANGUAGE_ENV, "sw_KE")
    assert W.resolve_colbert(p) is None
    with pytest.raises(ValueError, match="model_type 'xmod' is not supported in language 'sw_KE'"):
        W.resolve_model(p, with_head=True)
    monkeypatch.delenv(W.XMOD_LANGUAGE_ENV)
    with open(os.path.join(p, "config.json")) as f:
        conf = json.load(f)
    with open(os.path.join(p, "config.json"), "w") as f:
        json.dump({**conf, "default_language": None}, f)
    assert W.resolve_colbert(p) is None
    with pytest.raises(ValueError, match="model_type 'xmod' is not supported without an input language"):
        W.resolve_model(p, with_head=True)
    # an XLM-R model_type with the encoder under bert. contradicts itself
    q = _colbert_snapshot(tmp_path / "mixed", cfg, w, lin, kind="roberta", prefix="bert.")
    with pytest.raises(ValueError, match="under 'bert.'"):
        W.resolve_colbert(q)
    # an XLM-R ColBERT, bare tensor names
    xcfg = W.XLMRConfig(vocab_size=2000, hidden=256, layers=2, heads=4, ffn=512, max_pos=130)
    xw = synthetic_bert_weights(xcfg, seed=4)
    for kind in ("xlm-roberta", "roberta"):
        got = W.resolve_colbert(_colbert_snapshot(tmp_path / kind, xcfg, xw, lin, kind=kind, prefix=""))
        assert type(got[0]) is W.XLMRConfig and got[0].adapter_dim == 0
    # MPNet is refused
    q = _colbert_snapshot(tmp_path / "mp", xcfg, xw, lin, kind="mpnet", prefix="")
    with pytest.raises(ValueError, match="model_type 'mpnet' is not supported"):
        W.resolve_colbert(q)


def test_flashrank_refuses_xmod():
    with pytest.raises(ValueError, match="X-MOD"):
        W.resolve_flashrank("synthetic:tiny-xmod")


def test_presets_and_synthetic_weights():
    for name, A in (("xmod-base", 384), ("tiny-xmod", 128)):
        cfg = PRESETS[name][0]
        assert isinstance(cfg, XmodConfig) and cfg.adapter_dim == A and len(cfg.languages) >= 3
    cb = W.COLBERT_PRESETS["colbert-xm"]
    assert asdict(cb[0]) == asdict(PRESETS["xmod-base"][0]) and (cb[1].dim, cb[1].query_maxlen, cb[1].doc_maxlen) == (128, 32, 220)
    t = PRESETS["tiny-xmod"][0]
    assert (t.hidden, t.layers, t.heads, t.ffn, t.vocab_size, t.max_pos) == (256, 2, 4, 512, 2000, 130)
    cfg = _cfg()
    w = synthetic_bert_weights(cfg, seed=5)
    for lang in cfg.languages:                                          # an adapter set for every language
        for l in range(cfg.layers):
            for n, shape in W.adapter_names(cfg, l, lang):
                assert w[n].shape == shape
    # the rest of the weights are the XLM-R config's of the same shape and seed
    x = synthetic_bert_weights(W.XLMRConfig(**{k: v for k, v in asdict(cfg).items()
                                               if k not in ("adapter_dim", "languages", "language")}), seed=5)
    assert all(np.array_equal(x[k], w[k]) for k in x)


# ----------------------------------------------------------------------------------------------------------- C ABI
def test_config_struct_field():
    from ragmeup_b200 import _lib
    assert _lib.BertConfigC._fields_[-1] == ("adapter_dim", ctypes.c_int32)
    assert ctypes.sizeof(_lib.BertConfigC) == 12 * 4
    assert _lib.bert_config_c(_cfg()).adapter_dim == 128
    assert _lib.bert_config_c(W.BertConfig()).adapter_dim == 0
    assert _lib.bert_config_c(W.XLMRConfig()).adapter_dim == 0


def _create(cfg, arrs, has_head=0):
    from ragmeup_b200 import _lib
    ptrs = (ctypes.c_void_p * len(arrs))(*[None if a is None else a.ctypes.data for a in arrs])
    cc = _lib.bert_config_c(cfg)
    h = ctypes.c_void_p()
    rc = _lib.lib().rmu_encoder_create(ctypes.byref(cc), ptrs, len(arrs), has_head, ctypes.byref(h))
    if rc == 0:
        _lib.lib().rmu_encoder_destroy(h)
    return rc


def test_abi_adapter_refusals_before_any_cuda_call():
    cfg = _cfg()
    w = synthetic_bert_weights(cfg, seed=0, with_head=True)
    arrs = [np.ascontiguousarray(w[n]) for n, _ in weight_names(cfg, True)]
    for A in (64, 100, -128, 640):                                     # not a multiple of 128, or above ffn = 512
        assert _create(_cfg(adapter_dim=A), arrs, 1) == -3, A
    assert _create(cfg, arrs[:-1], 1) == -1                            # one adapter tensor missing
    assert _create(cfg, arrs[:-1] + [None], 1) == -1                   # a null adapter tensor
    assert _create(_cfg(adapter_dim=0), arrs, 1) == -1                 # the adapters with adapter_dim = 0
    big = [a.copy() for a in arrs]
    big[-2].reshape(-1)[7] = 70000.0                                   # the last adapter's dense2 weight
    assert _create(cfg, big, 1) == -3
    from ragmeup_b200 import _lib
    assert "adapter dense2" in _lib.lib().rmu_last_error().decode()
    assert _create(cfg, arrs, 1) in (0, -2)                            # accepted: without a device the next step fails
