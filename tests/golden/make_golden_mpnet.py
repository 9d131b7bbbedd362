"""Mint tests/golden/mpnet.npz from ``transformers.MPNetModel`` (attn_implementation="eager", fp32) fed the seeded
synthetic weights the tests rebuild with ``ragmeup_b200.weights.synthetic_bert_weights``; only token ids and outputs
are stored.  Separate from make_golden.py, so the other golden files are not rewritten.

Usage:  python tests/golden/make_golden_mpnet.py
"""
import os
import sys
from dataclasses import asdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from ragmeup_b200.weights import PRESETS, MPNetConfig, synthetic_bert_weights  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# (preset, seed, scale, lengths, sequence holding id 1 mid-text or None)
CASES = [("all-mpnet-base-v2", 0, 1.0, [1, 9, 16, 129, 384, 512], 3),
         ("tiny-mpnet", 2, 4.0, [1, 9, 16, 64, 128, 5], 4)]


def hf_state_dict(w):
    """canonical (BERT) names -> MPNetModel's"""
    ren = (("attention.self.query.", "attention.attn.q."), ("attention.self.key.", "attention.attn.k."),
           ("attention.self.value.", "attention.attn.v."), ("attention.output.dense.", "attention.attn.o."),
           ("attention.output.LayerNorm.", "attention.LayerNorm."))
    sd = {}
    for k, v in w.items():
        if k == "embeddings.token_type_embeddings.weight":
            continue
        for a, b in ren:
            k = k.replace(a, b)
        sd[k] = torch.from_numpy(v)
    return sd


def hf_model(cfg: MPNetConfig, w):
    from transformers import MPNetConfig as HC, MPNetModel
    hc = HC(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, num_hidden_layers=cfg.layers,
            num_attention_heads=cfg.heads, intermediate_size=cfg.ffn, max_position_embeddings=cfg.max_pos,
            layer_norm_eps=cfg.ln_eps, relative_attention_num_buckets=32, hidden_dropout_prob=0.0,
            attention_probs_dropout_prob=0.0, attn_implementation="eager")
    m = MPNetModel(hc, add_pooling_layer=False).eval()
    missing = m.load_state_dict(hf_state_dict(w), strict=False)
    bad = [k for k in missing.missing_keys if "position_ids" not in k]
    assert not bad and not missing.unexpected_keys, (bad, missing.unexpected_keys)
    return m


def batch(rng, cfg, lens, pad_seq):
    """<s> ... </s> sequences padded with <pad> = 1; sequence pad_seq holds id 1 at a third and at two thirds of it"""
    B, S = len(lens), max(lens)
    ids = np.ones((B, S), dtype=np.int64)
    mask = np.zeros((B, S), dtype=np.int64)
    for b, n in enumerate(lens):
        ids[b, :n] = rng.integers(5, cfg.vocab_size - 1, n)
        ids[b, 0] = 0
        ids[b, n - 1] = 2
        mask[b, :n] = 1
    if pad_seq is not None:
        n = lens[pad_seq]
        ids[pad_seq, n // 3] = 1
        ids[pad_seq, 2 * n // 3] = 1
    return ids, mask


def mpnet_goldens():
    rng = np.random.default_rng(2024)
    out = {}
    for preset, seed, scale, lens, pad_seq in CASES:
        cfg = MPNetConfig(**asdict(PRESETS[preset][0]))
        w = synthetic_bert_weights(cfg, seed=seed, with_head=False, scale=scale)
        m = hf_model(cfg, w)
        ids, mask = batch(rng, cfg, lens, pad_seq)
        with torch.no_grad():
            h = m(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask)).last_hidden_state
        mk = torch.from_numpy(mask)[..., None].float()
        mean = torch.nn.functional.normalize((h * mk).sum(1) / mk.sum(1).clamp(min=1e-9), p=2, dim=1)
        key = f"mpnet_{preset}_{seed}_{scale}"
        out[key + "_ids"] = ids.astype(np.int32)
        out[key + "_mask"] = mask.astype(np.int8)
        out[key + "_mean"] = mean.numpy()
        out[key + "_cls"] = torch.nn.functional.normalize(h[:, 0], p=2, dim=1).numpy()
        out[key + "_h_first"] = h[:, 0].numpy()
        out[key + "_h_last"] = np.stack([h[b, n - 1].numpy() for b, n in enumerate(lens)])
    return out


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    np.savez_compressed(os.path.join(HERE, "mpnet.npz"), **mpnet_goldens())
    print("mpnet.npz", os.path.getsize(os.path.join(HERE, "mpnet.npz")) // 1024, "KiB")
