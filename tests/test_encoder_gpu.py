"""GPU parity: BERT encoder / cross-encoder through the C ABI vs the goldens (HF transformers) and
the oracle.  Tolerance 1e-3 on embeddings and logits (BASELINE.json)."""
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import bert_ref
from ragmeup_b200.weights import PRESETS, BertConfig, synthetic_bert_weights

pytestmark = pytest.mark.gpu
TOL = 1e-3
ENC_CASES = [("tiny", 0, 1.0), ("all-MiniLM-L6-v2", 0, 1.0), ("all-MiniLM-L6-v2", 1, 4.0), ("bge-base-en-v1.5", 0, 1.0)]
CE_CASES = [("tiny", 3, 4.0), ("ms-marco-MiniLM-L-6-v2", 0, 1.0), ("ms-marco-MiniLM-L-6-v2", 2, 6.0)]


def _ragged(ids, mask, typ):
    lens = mask.sum(1)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    rid = np.concatenate([ids[b, :n] for b, n in enumerate(lens)]).astype(np.int32)
    rty = np.concatenate([typ[b, :n] for b, n in enumerate(lens)]).astype(np.int32)
    return rid, rty, cu, int(lens.max())


@pytest.mark.parametrize("preset,seed,scale", ENC_CASES)
def test_embeddings_match_hf_golden(cuda, golden_dir, preset, seed, scale):
    from ragmeup_b200.encoder import BertEncoder
    g = np.load(f"{golden_dir}/encoder.npz")
    key = f"enc_{preset}_{seed}_{scale}"
    cfg = BertConfig(**asdict(PRESETS[preset][0]))
    enc = BertEncoder(cfg, synthetic_bert_weights(cfg, seed=seed, scale=scale), with_head=False)
    ids, typ, cu, mx = _ragged(g[key + "_ids"].astype(np.int64), g[key + "_mask"].astype(np.int64), g[key + "_typ"].astype(np.int64))
    mean = enc.embed_tokens(ids, typ, cu, mx, "mean", True).cpu().numpy()
    cls = enc.embed_tokens(ids, typ, cu, mx, "cls", True).cpu().numpy()
    assert np.abs(mean - g[key + "_mean"]).max() < TOL
    assert np.abs(cls - g[key + "_cls"]).max() < TOL
    h = enc.hidden_tokens(ids, typ, cu, mx).cpu().numpy()
    assert np.abs(h[cu[:-1]] - g[key + "_h_first"]).max() < 5e-3
    assert np.abs(h[cu[1:] - 1] - g[key + "_h_last"]).max() < 5e-3
    # host-buffer entry point returns the same numbers
    assert np.abs(enc.embed_host(ids, typ, cu, "mean", True) - mean).max() < 1e-6
    # unnormalised mean pooling
    raw = enc.embed_tokens(ids, typ, cu, mx, "mean", False).cpu().numpy()
    assert np.abs(raw / np.linalg.norm(raw, axis=1, keepdims=True) - mean).max() < 1e-5


@pytest.mark.parametrize("preset,seed,scale", CE_CASES)
def test_logits_match_hf_golden(cuda, golden_dir, preset, seed, scale):
    from ragmeup_b200.encoder import BertEncoder
    g = np.load(f"{golden_dir}/cross_encoder.npz")
    key = f"ce_{preset}_{seed}_{scale}"
    cfg = BertConfig(**asdict(PRESETS[preset][0]))
    enc = BertEncoder(cfg, synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale), with_head=True)
    ids, typ, cu, mx = _ragged(g[key + "_ids"].astype(np.int64), g[key + "_mask"].astype(np.int64), g[key + "_typ"].astype(np.int64))
    lg = enc.classify_tokens(ids, typ, cu, mx).cpu().numpy()
    assert np.abs(lg - g[key + "_logits"]).max() < TOL
    assert np.abs(enc.classify_host(ids, typ, cu) - lg).max() < 1e-6


def test_ragged_batch_vs_oracle_long_sequences(cuda):
    """S up to 512 (truncation limit), 150-token rerank-shaped pairs, single-token edge"""
    from ragmeup_b200.encoder import BertEncoder
    preset = "ms-marco-MiniLM-L-6-v2"
    cfg = BertConfig(**asdict(PRESETS[preset][0]))
    ocfg = bert_ref.BertCfg(**asdict(cfg))
    w = synthetic_bert_weights(cfg, seed=5, with_head=True, scale=4.0)
    enc = BertEncoder(cfg, w, with_head=True)
    rng = np.random.default_rng(9)
    lens = [512, 147, 147, 2, 300, 31]
    ids = np.concatenate([np.r_[101, rng.integers(104, cfg.vocab_size, n - 2), 102] for n in lens]).astype(np.int32)
    typ = np.concatenate([np.r_[np.zeros(n // 3, np.int32), np.ones(n - n // 3, np.int32)] for n in lens])
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    lg = enc.classify_tokens(ids, typ, cu, max(lens)).cpu()
    S = max(lens)
    I = np.zeros((len(lens), S), np.int64); M = np.zeros_like(I); T = np.zeros_like(I)
    for b, n in enumerate(lens):
        I[b, :n] = ids[cu[b]:cu[b + 1]]; T[b, :n] = typ[cu[b]:cu[b + 1]]; M[b, :n] = 1
    with torch.no_grad():
        h = bert_ref.bert_encoder_forward(w, ocfg, torch.from_numpy(I), torch.from_numpy(M), torch.from_numpy(T))
        ref = bert_ref.classifier_head(w, h)
    assert float((lg - ref).abs().max()) < TOL
    # batch-composition invariance: each sequence alone gives the same logit
    for b in (1, 3):
        one = enc.classify_tokens(ids[cu[b]:cu[b + 1]], typ[cu[b]:cu[b + 1]], np.array([0, lens[b]], np.int32), lens[b]).cpu()
        assert float((one[0] - lg[b]).abs().max()) < 1e-5


def _oracle_hidden(w, cfg, ids, typ, lens):
    cu = np.r_[0, np.cumsum(lens)]
    S = max(lens)
    I = np.zeros((len(lens), S), np.int64); M = np.zeros_like(I); T = np.zeros_like(I)
    for b, n in enumerate(lens):
        I[b, :n] = ids[cu[b]:cu[b + 1]]; T[b, :n] = typ[cu[b]:cu[b + 1]]; M[b, :n] = 1
    with torch.no_grad():
        h = bert_ref.bert_encoder_forward(w, bert_ref.BertCfg(**asdict(cfg)), torch.from_numpy(I), torch.from_numpy(M),
                                          torch.from_numpy(T))
    return h, torch.from_numpy(M)


@pytest.mark.parametrize("preset,lens", [
    # d_h = 64, K = 768 and 3072; 160-row blocks past the first, the 256-key super-block, a 1-token sequence
    ("bge-base-en-v1.5", [512, 300, 257, 161, 33, 1]),
    # K = 128 and 256 with 9 000 tokens: 213 QKV and 142 FFN-in tiles on 132 SMs, so both consumer warpgroups of a
    # CTA run and the ring starts a tile at every slot
    ("tiny", [int(n) for n in np.random.default_rng(11).integers(110, 129, 75)]),
])
def test_encoder_matches_oracle_at_scale(cuda, preset, lens):
    from ragmeup_b200.encoder import BertEncoder
    cfg = BertConfig(**asdict(PRESETS[preset][0]))
    w = synthetic_bert_weights(cfg, seed=21, scale=1.0)
    enc = BertEncoder(cfg, w, with_head=False)
    rng = np.random.default_rng(12)
    ids = np.concatenate([np.r_[101, rng.integers(104, cfg.vocab_size, max(n - 2, 0)), 102][:n] for n in lens]).astype(np.int32)
    typ = np.concatenate([np.r_[np.zeros(n // 2, np.int32), np.ones(n - n // 2, np.int32)] for n in lens])
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    href, mask = _oracle_hidden(w, cfg, ids, typ, lens)
    h = enc.hidden_tokens(ids, typ, cu, max(lens)).cpu()
    flat = torch.cat([href[b, :n] for b, n in enumerate(lens)])
    herr = float((h - flat).abs().max())
    for mode in ("mean", "cls"):
        e = enc.embed_tokens(ids, typ, cu, max(lens), mode, True).cpu()
        want = bert_ref.l2_normalize(bert_ref.pool(href, mask, mode))
        eerr = float((e - want).abs().max())
        print(f"\n{preset} T={cu[-1]}: hidden max err {herr:.3g}, {mode} embedding max err {eerr:.3g}")
        assert eerr < TOL
    assert herr < 5e-3          # the hidden-state bound of test_embeddings_match_hf_golden
