"""Mint tests/golden/xlmr.npz from ``transformers.XLMRobertaModel`` and ``XLMRobertaForSequenceClassification``
(attn_implementation="eager", fp32) fed the seeded synthetic weights the tests rebuild with
``ragmeup_b200.weights.synthetic_bert_weights``; only token ids and outputs are stored.  Separate from make_golden.py
and make_golden_mpnet.py, so the other golden files are not rewritten.

Usage:  python tests/golden/make_golden_xlmr.py
"""
import os
import sys
from dataclasses import asdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from ragmeup_b200.weights import PRESETS, XLMRConfig, synthetic_bert_weights  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# (preset, seed, scale, with the classification head, lengths, sequence holding id 1 mid-text or None)
CASES = [("bge-reranker-base", 0, 1.0, True, [1, 9, 16, 129, 384, 512], 3),
         ("tiny-xlmr", 2, 4.0, True, [1, 9, 16, 64, 128, 5], 4),
         ("tiny-xlmr-long", 1, 1.0, False, [3, 513, 1500, 40], 2)]


def hf_state_dict(w, head: bool):
    """canonical names -> XLMRobertaModel's (bare) or XLMRobertaForSequenceClassification's (under roberta., with the
    head as classifier.dense / classifier.out_proj)"""
    sd = {}
    for k, v in w.items():
        if k.startswith("pooler.dense."):
            k = "classifier.dense." + k[13:]
        elif k.startswith("classifier."):
            k = "classifier.out_proj." + k[11:]
        elif head:
            k = "roberta." + k
        sd[k] = torch.from_numpy(v)
    return sd


def hf_model(cfg: XLMRConfig, w, head: bool):
    from transformers import XLMRobertaConfig as HC, XLMRobertaForSequenceClassification, XLMRobertaModel
    hc = HC(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, num_hidden_layers=cfg.layers,
            num_attention_heads=cfg.heads, intermediate_size=cfg.ffn, max_position_embeddings=cfg.max_pos,
            type_vocab_size=1, layer_norm_eps=cfg.ln_eps, pad_token_id=1, num_labels=cfg.num_labels,
            hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, attn_implementation="eager")
    m = (XLMRobertaForSequenceClassification(hc) if head else XLMRobertaModel(hc, add_pooling_layer=False)).eval()
    res = m.load_state_dict(hf_state_dict(w, head), strict=False)
    bad = [k for k in res.missing_keys if "position_ids" not in k]
    assert not bad and not res.unexpected_keys, (bad, res.unexpected_keys)
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


def xlmr_goldens():
    rng = np.random.default_rng(2025)
    out = {}
    for preset, seed, scale, head, lens, pad_seq in CASES:
        cfg = XLMRConfig(**asdict(PRESETS[preset][0]))
        w = synthetic_bert_weights(cfg, seed=seed, with_head=head, scale=scale)
        m = hf_model(cfg, w, head)
        ids, mask = batch(rng, cfg, lens, pad_seq)
        with torch.no_grad():
            r = m(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), output_hidden_states=True)
        h = r.hidden_states[-1]
        mk = torch.from_numpy(mask)[..., None].float()
        key = f"xlmr_{preset}_{seed}_{scale}"
        out[key + "_ids"] = ids.astype(np.int32)
        out[key + "_mask"] = mask.astype(np.int8)
        out[key + "_mean"] = torch.nn.functional.normalize((h * mk).sum(1) / mk.sum(1).clamp(min=1e-9), p=2, dim=1).numpy()
        out[key + "_cls"] = torch.nn.functional.normalize(h[:, 0], p=2, dim=1).numpy()
        out[key + "_h_first"] = h[:, 0].numpy()
        out[key + "_h_last"] = np.stack([h[b, n - 1].numpy() for b, n in enumerate(lens)])
        if head:
            out[key + "_logits"] = r.logits.numpy()
    return out


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    np.savez_compressed(os.path.join(HERE, "xlmr.npz"), **xlmr_goldens())
    print("xlmr.npz", os.path.getsize(os.path.join(HERE, "xlmr.npz")) // 1024, "KiB")
