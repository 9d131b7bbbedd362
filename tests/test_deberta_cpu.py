"""CPU: DeBERTa-v3 cross-encoders (mixedbread-ai/mxbai-rerank-*-v1).  The fp32 and float64 oracles against the goldens
minted from transformers' DebertaV2ForSequenceClassification (tests/golden/make_golden_deberta.py); the host bucket
table against make_log_bucket_position; the p2c index identity; every refusal; a save_pretrained snapshot; PairAssembler
against pair tokenisation on a DeBERTa-shaped tokenizer; and rmu_encoder_create_ex's refusals without a device."""
import ctypes
import json
import os
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import deberta_ref
from ragmeup_b200 import weights as W
from ragmeup_b200.weights import PRESETS, DebertaConfig, synthetic_bert_weights, weight_names

GOLDEN = [(0, 1.0), (3, 4.0)]


def _cfg(preset="tiny-deberta"):
    return DebertaConfig(**asdict(PRESETS[preset][0]))


@pytest.mark.parametrize("seed,scale", GOLDEN)
def test_deberta_oracle_matches_hf(golden_dir, seed, scale):
    """fp32 forward (padded) and float64 ragged stack against transformers, lengths across |i - j| = 128 up to 512"""
    g = np.load(f"{golden_dir}/deberta.npz")
    key = f"deberta_tiny-deberta_{seed}_{scale}"
    cfg = _cfg()
    w = synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale)
    ids = torch.from_numpy(g[key + "_ids"].astype(np.int64))
    mask = torch.from_numpy(g[key + "_mask"].astype(np.int64))
    lens = mask.sum(1).tolist()
    assert max(lens) == 512 or max(lens) > 256
    with torch.no_grad():
        h = deberta_ref.deberta_encoder_forward(w, cfg, ids, mask)
        logits = deberta_ref.classifier_head(w, h).numpy()
    tol = 4e-6 if scale == 1.0 else 2e-5
    want = g[key + "_logits"]
    assert np.abs(h[:, 0].numpy() - g[key + "_h_first"]).max() < 50 * tol
    assert np.abs(logits - want).max() < 50 * tol * max(1.0, float(np.abs(want).max()))
    flat = np.concatenate([g[key + "_ids"][b, :n] for b, n in enumerate(lens)])
    cu = np.r_[0, np.cumsum(lens)]
    ref = deberta_ref.deberta_stack_ref(w, cfg, flat, cu)
    assert float((ref["hidden"][cu[1:] - 1] - torch.from_numpy(g[key + "_h_last"]).double()).abs().max()) < 50 * tol
    assert float((ref["logits"] - torch.from_numpy(want).double()).abs().max()) < 50 * tol * max(1.0, float(np.abs(want).max()))


def _host_buckets(s, max_position, n):
    from ragmeup_b200 import _lib
    out = np.zeros(2 * n - 1, np.int32)
    _lib.check(_lib.lib().rmu_log_bucket_table(s, max_position, n, out.ctypes.data), "rmu_log_bucket_table")
    return out


@pytest.mark.parametrize("s,max_position,n", [(256, 512, 512), (128, 512, 512), (64, 300, 300), (256, 1024, 1024)])
def test_host_bucket_table_equals_make_log_bucket_position(s, max_position, n):
    from transformers.models.deberta_v2.modeling_deberta_v2 import make_log_bucket_position
    r = torch.arange(-(n - 1), n)
    want = make_log_bucket_position(r, s, max_position).long().numpy()
    assert np.array_equal(_host_buckets(s, max_position, n), want)
    assert np.array_equal(deberta_ref.log_bucket(r.numpy(), s, max_position), want)


def test_clamp_never_bites_within_512_tokens():
    """s = 256, max_position 512: |r| <= 511 gives c in [1, 511]"""
    c = 256 + _host_buckets(256, 512, 512)
    assert c.min() == 1 and c.max() == 511


def test_p2c_index_identity():
    """transformers gathers p2c at s - bucket(j - i) and transposes: that is s + bucket(i - j), bucket being odd"""
    from transformers.models.deberta_v2.modeling_deberta_v2 import build_relative_position
    S, s = 300, 256
    q = torch.zeros(1, S, 1)
    rel = build_relative_position(q, q, bucket_size=s, max_position=512).long().reshape(S, S)
    idx_p2c = torch.clamp(-rel + s, 0, 2 * s - 1)            # [a, b], read transposed: score(i, j) uses [j, i]
    want = torch.from_numpy(deberta_ref.position_index(S, s, 512))
    assert torch.equal(idx_p2c.t(), want)
    assert torch.equal(torch.clamp(rel + s, 0, 2 * s - 1), want)        # c2p


# ------------------------------------------------------------------------------------------------- config, snapshots
BASE = dict(model_type="deberta-v2", vocab_size=2000, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
            intermediate_size=256, max_position_embeddings=512, relative_attention=True, position_buckets=256,
            share_att_key=True, pos_att_type=["p2c", "c2p"], norm_rel_ebd="layer_norm", position_biased_input=False,
            type_vocab_size=0, hidden_act="gelu", pooler_hidden_act="gelu", layer_norm_eps=1e-7,
            max_relative_positions=-1)


@pytest.mark.parametrize("field,value", [("relative_attention", False), ("position_buckets", 0),
                                         ("position_buckets", -1), ("share_att_key", False),
                                         ("pos_att_type", ["c2p"]), ("pos_att_type", "p2c|c2p|p2p"),
                                         ("norm_rel_ebd", "none"), ("position_biased_input", True),
                                         ("type_vocab_size", 2), ("conv_kernel_size", 3), ("embedding_size", 256),
                                         ("hidden_act", "gelu_new"), ("pooler_hidden_act", "tanh")])
def test_config_refusals_name_the_field(field, value):
    with pytest.raises(ValueError, match=field):
        DebertaConfig.from_hf({**BASE, field: value})


def test_config_reads_fields():
    c = DebertaConfig.from_hf({**BASE, "pos_att_type": "p2c|c2p"})
    assert (c.position_buckets, c.max_relative_positions, c.head_act, c.max_pos, c.type_vocab) == (256, 512, 1, 512, 1)
    assert DebertaConfig.from_hf({**BASE, "max_relative_positions": 300}).max_relative_positions == 300


def _hf_model(num_labels=1):
    from transformers import DebertaV2Config, DebertaV2ForSequenceClassification
    torch.manual_seed(0)
    hc = DebertaV2Config(**{k: v for k, v in BASE.items() if k != "model_type"}, num_labels=num_labels,
                         pooler_hidden_size=128)
    return DebertaV2ForSequenceClassification(hc).eval()


def _save(m, path, tokenizer=True, spm=False, model_max_length=None):
    m.save_pretrained(path)
    if tokenizer:
        from ragmeup_b200.tokenizer import load_tokenizer
        load_tokenizer(None, m.config.vocab_size, deberta=True).save(os.path.join(path, "tokenizer.json"))
    if spm:
        open(os.path.join(path, "spm.model"), "wb").close()
    if model_max_length is not None:
        with open(os.path.join(path, "tokenizer_config.json"), "w") as f:
            json.dump({"model_max_length": model_max_length}, f)
    return path


def test_snapshot_from_save_pretrained(tmp_path):
    from ragmeup_b200.weights import resolve_model
    m = _hf_model()
    path = _save(m, str(tmp_path / "mxbai-rerank-base-v1"), model_max_length=256)
    cfg, w, _p, _n, max_len, act, src = resolve_model(path, with_head=True)
    assert isinstance(cfg, DebertaConfig) and (max_len, act, src, cfg.num_labels) == (256, "sigmoid", path, 1)
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    H = cfg.hidden
    for l in range(cfg.layers):
        for a in ("query", "key", "value"):
            for t in ("weight", "bias"):
                assert np.array_equal(w[f"encoder.layer.{l}.attention.self.{a}.{t}"],
                                      sd[f"deberta.encoder.layer.{l}.attention.self.{a}_proj.{t}"])
    assert np.array_equal(w["encoder.rel_embeddings.weight"], sd["deberta.encoder.rel_embeddings.weight"][:512])
    assert np.array_equal(w["encoder.LayerNorm.weight"], sd["deberta.encoder.LayerNorm.weight"])
    assert np.array_equal(w["pooler.dense.weight"], sd["pooler.dense.weight"])
    assert np.array_equal(w["classifier.bias"], sd["classifier.bias"])
    assert not w["embeddings.position_embeddings.weight"].any() and w["embeddings.position_embeddings.weight"].shape == (512, H)
    assert not w["embeddings.token_type_embeddings.weight"].any()
    names = [n for n, _ in weight_names(cfg, True)]
    assert names[-3:] == ["encoder.rel_embeddings.weight", "encoder.LayerNorm.weight", "encoder.LayerNorm.bias"]
    assert all(n in w for n in names)
    # the oracle on these tensors equals transformers' own forward
    ids = torch.tensor([[1, 50, 60, 70, 2, 80, 90, 2]])
    with torch.no_grad():
        want = m(input_ids=ids).logits.numpy()
        got = deberta_ref.classifier_head(w, deberta_ref.deberta_encoder_forward(w, cfg, ids, torch.ones_like(ids))).numpy()
    assert np.abs(got - want).max() < 1e-5


def test_snapshot_refusals(tmp_path):
    from ragmeup_b200.tokenizer import load_tokenizer
    from ragmeup_b200.weights import resolve_flashrank, resolve_model
    m = _hf_model()
    path = _save(m, str(tmp_path / "a"), tokenizer=False, spm=True)
    with pytest.raises(ValueError, match="spm.model"):
        load_tokenizer(path, 2000, deberta=True)
    with pytest.raises(ValueError, match="deberta-v2"):
        resolve_model(path, with_head=False)                  # HuggingFaceEmbeddings
    with pytest.raises(ValueError, match="deberta-v2"):
        resolve_model("synthetic:tiny-deberta", with_head=False)
    with pytest.raises(ValueError, match="DeBERTa"):
        resolve_flashrank("synthetic:tiny-deberta")
    with open(os.path.join(path, "config.json")) as f:
        conf = json.load(f)
    conf["model_type"] = "deberta"
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(conf, f)
    with pytest.raises(ValueError, match="'deberta'"):
        resolve_model(path, with_head=True)


def test_colbert_refuses_deberta(tmp_path):
    from ragmeup_b200.weights import load_colbert_snapshot
    path = tmp_path / "c"
    path.mkdir()
    with open(path / "config.json", "w") as f:
        json.dump(BASE, f)
    with pytest.raises(ValueError, match="deberta-v2"):
        load_colbert_snapshot(str(path))


def test_tokens_per_call_bounds_the_workspace():
    from ragmeup_b200.encoder import MAX_TOKENS_PER_CALL, POSITION_WS_BYTES, deberta_tokens_per_call
    for p in ("mxbai-rerank-xsmall-v1", "mxbai-rerank-base-v1", "mxbai-rerank-large-v1", "tiny-deberta"):
        c = _cfg(p)
        n = deberta_tokens_per_call(c)
        assert n * 2 * c.heads * 2 * c.position_buckets * 4 <= POSITION_WS_BYTES and n >= 512
    assert deberta_tokens_per_call(W.BertConfig()) == MAX_TOKENS_PER_CALL


# ------------------------------------------------------------------------------------------------- tokenisation
def test_pair_assembler_equals_pair_tokenisation():
    from ragmeup_b200.tokenizer import PairAssembler, RaggedTokenizer, load_tokenizer
    tok = load_tokenizer(None, 2000, deberta=True)
    e = tok.encode("ba ce", "di")
    assert e.ids[0] == 1 and e.ids[-1] == 2 and e.type_ids[0] == 0 and e.type_ids[-1] == 1
    rng = np.random.default_rng(0)
    syl = ["ba", "ce", "di", "fo", "gu", "ha", "je", "ki", "lo", "mu", "[SEP]", "x", ",", "  "]
    texts = [" ".join("".join(syl[j] for j in rng.integers(0, len(syl), 3)) for _ in range(int(rng.integers(0, 200))))
             for _ in range(60)]
    a, b = texts[:30], texts[30:]
    for max_len in (512, 64, 7):
        got = PairAssembler(tok, max_len)(a, b)
        want = RaggedTokenizer(tok, max_len)(a, b)
        for x, y in zip(got, want):
            assert np.array_equal(x, y)


# ------------------------------------------------------------------------------------------------- C refusals
def _create(cfg, arrs, ext=None, has_head=1):
    from ragmeup_b200 import _lib
    ptrs = (ctypes.c_void_p * len(arrs))(*[None if a is None else a.ctypes.data for a in arrs])
    cc = _lib.bert_config_c(cfg)
    ex = ext if ext is not None else _lib.encoder_ext_c(cfg)
    h = ctypes.c_void_p()
    return _lib.lib().rmu_encoder_create_ex(ctypes.byref(cc), ctypes.byref(ex), ptrs, len(arrs), has_head, ctypes.byref(h))


def test_create_refuses_bad_fields_without_a_device():
    from ragmeup_b200 import _lib
    cfg = _cfg()
    w = synthetic_bert_weights(cfg, seed=0, with_head=True)
    arrs = [w[n] for n, _ in weight_names(cfg, True)]
    E = _lib.EncoderExtC
    for ext, rc in ((E(256, 512, 2), -3), (E(-1, 0, 1), -3), (E(0, 512, 1), -3), (E(256, 129, 1), -3),
                    (E(8192, 8192, 1), -3), (E(1, 3, 1), -3)):
        assert _create(cfg, arrs, ext) == rc, (ext.position_buckets, ext.max_relative_positions, ext.head_act)
    assert _create(cfg, arrs[:-1]) == -1                     # LN_rel's bias missing
    assert _create(cfg, arrs[:-3] + [None, arrs[-2], arrs[-1]]) == -1
    assert "relative embedding" in _lib.lib().rmu_last_error().decode()
    bad = DebertaConfig(**{**asdict(cfg), "hidden": 128, "heads": 4})            # head_dim 32
    assert _create(bad, arrs) == -3
    assert "head_dim 64" in _lib.lib().rmu_last_error().decode()
    assert _lib.lib().rmu_log_bucket_table(256, 100, 10, np.zeros(19, np.int32).ctypes.data) == -3
