"""Mint tests/golden/deberta.npz from ``transformers.DebertaV2ForSequenceClassification`` (attn_implementation="eager",
fp32) fed the seeded synthetic weights the tests rebuild with ``ragmeup_b200.weights.synthetic_bert_weights``; only
token ids, masks and outputs are stored.  The lengths cross |i - j| = 128 (the end of the exact buckets with s = 256)
and reach 512.  Separate from the other generators, so their golden files are not rewritten.

Usage:  python tests/golden/make_golden_deberta.py
"""
import os
import sys
from dataclasses import asdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from ragmeup_b200.weights import PRESETS, DebertaConfig, synthetic_bert_weights  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# (preset, seed, scale, lengths)
CASES = [("tiny-deberta", 0, 1.0, [1, 9, 127, 130, 300, 512]),
         ("tiny-deberta", 3, 4.0, [2, 64, 129, 257, 200])]


def hf_config(cfg: DebertaConfig, **kw):
    from transformers import DebertaV2Config
    return DebertaV2Config(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, num_hidden_layers=cfg.layers,
                           num_attention_heads=cfg.heads, intermediate_size=cfg.ffn,
                           max_position_embeddings=cfg.max_pos, type_vocab_size=0, layer_norm_eps=cfg.ln_eps,
                           relative_attention=True, position_buckets=cfg.position_buckets, norm_rel_ebd="layer_norm",
                           share_att_key=True, pos_att_type=["p2c", "c2p"], position_biased_input=False,
                           max_relative_positions=-1, hidden_act="gelu", pooler_hidden_act="gelu",
                           pooler_hidden_size=cfg.hidden, num_labels=cfg.num_labels, hidden_dropout_prob=0.0,
                           attention_probs_dropout_prob=0.0, pooler_dropout=0.0, attn_implementation="eager", **kw)


def hf_state_dict(w):
    """canonical names -> DebertaV2ForSequenceClassification's (under deberta., the head bare); the zero position
    and token-type tables have no counterpart"""
    sd = {}
    for k, v in w.items():
        if k in ("embeddings.position_embeddings.weight", "embeddings.token_type_embeddings.weight"):
            continue
        if k.startswith(("pooler.", "classifier.")):
            sd[k] = torch.from_numpy(v)
            continue
        for a in ("query", "key", "value"):
            k = k.replace(f"attention.self.{a}.", f"attention.self.{a}_proj.")
        sd["deberta." + k] = torch.from_numpy(v)
    return sd


def hf_model(cfg: DebertaConfig, w):
    from transformers import DebertaV2ForSequenceClassification
    m = DebertaV2ForSequenceClassification(hf_config(cfg)).eval()
    res = m.load_state_dict(hf_state_dict(w), strict=False)
    bad = [k for k in res.missing_keys if "position_ids" not in k]
    assert not bad and not res.unexpected_keys, (bad, res.unexpected_keys)
    return m


def batch(rng, cfg, lens):
    """[CLS] ... [SEP] sequences padded with [PAD] = 0"""
    B, S = len(lens), max(lens)
    ids = np.zeros((B, S), dtype=np.int64)
    mask = np.zeros((B, S), dtype=np.int64)
    for b, n in enumerate(lens):
        ids[b, :n] = rng.integers(4, cfg.vocab_size - 1, n)
        ids[b, 0] = 1
        ids[b, n - 1] = 2
        mask[b, :n] = 1
    return ids, mask


def deberta_goldens():
    rng = np.random.default_rng(2026)
    out = {}
    for preset, seed, scale, lens in CASES:
        cfg = DebertaConfig(**asdict(PRESETS[preset][0]))
        w = synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale)
        m = hf_model(cfg, w)
        ids, mask = batch(rng, cfg, lens)
        with torch.no_grad():
            r = m(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), output_hidden_states=True)
        h = r.hidden_states[-1]
        key = f"deberta_{preset}_{seed}_{scale}"
        out[key + "_ids"] = ids.astype(np.int32)
        out[key + "_mask"] = mask.astype(np.int8)
        out[key + "_h_first"] = h[:, 0].numpy()
        out[key + "_h_last"] = np.stack([h[b, n - 1].numpy() for b, n in enumerate(lens)])
        out[key + "_logits"] = r.logits.numpy()
    return out


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    np.savez_compressed(os.path.join(HERE, "deberta.npz"), **deberta_goldens())
    print("deberta.npz", os.path.getsize(os.path.join(HERE, "deberta.npz")) // 1024, "KiB")
