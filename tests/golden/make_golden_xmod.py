"""Mint tests/golden/xmod.npz from ``transformers.XmodModel`` and ``XmodForSequenceClassification``
(attn_implementation="eager", fp32) fed the seeded synthetic weights the tests rebuild with
``ragmeup_b200.weights.synthetic_bert_weights`` (an adapter set for each of three languages).  The model runs the
third language, which is neither the first nor config.default_language, so an oracle that took either would not match.
Only token ids and outputs are stored.  Separate from the other generators, so their golden files are not rewritten.

Usage:  python tests/golden/make_golden_xmod.py
"""
import os
import sys
from dataclasses import asdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from ragmeup_b200.weights import PRESETS, XmodConfig, synthetic_bert_weights  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_xlmr import batch, hf_state_dict  # noqa: E402

LANGUAGES = ("en_XX", "de_DE", "fr_XX")
DEFAULT, RUN = "de_DE", "fr_XX"
# (preset, seed, scale, lengths, sequence holding id 1 mid-text)
CASES = [("tiny-xmod", 0, 1.0, [1, 9, 16, 64, 128, 5], 3),
         ("tiny-xmod", 2, 4.0, [3, 40, 128, 2], 1)]


def xmod_cfg(preset) -> XmodConfig:
    return XmodConfig(**{**asdict(PRESETS[preset][0]), "languages": LANGUAGES, "language": RUN})


def hf_model(cfg: XmodConfig, w, head: bool, default_language=DEFAULT):
    from transformers import XmodConfig as HC, XmodForSequenceClassification, XmodModel
    hc = HC(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, num_hidden_layers=cfg.layers,
            num_attention_heads=cfg.heads, intermediate_size=cfg.ffn, max_position_embeddings=cfg.max_pos,
            type_vocab_size=1, layer_norm_eps=cfg.ln_eps, pad_token_id=1, num_labels=cfg.num_labels,
            hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, attn_implementation="eager",
            adapter_reduction_factor=cfg.hidden // cfg.adapter_dim, languages=list(cfg.languages),
            default_language=default_language)
    m = (XmodForSequenceClassification(hc) if head else XmodModel(hc, add_pooling_layer=False)).eval()
    res = m.load_state_dict(hf_state_dict(w, head), strict=False)
    bad = [k for k in res.missing_keys if "position_ids" not in k]
    assert not bad and not res.unexpected_keys, (bad, res.unexpected_keys)
    return m


def xmod_goldens():
    rng = np.random.default_rng(2026)
    out = {}
    for preset, seed, scale, lens, pad_seq in CASES:
        cfg = xmod_cfg(preset)
        w = synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale)
        m = hf_model(cfg, w, True)
        ids, mask = batch(rng, cfg, lens, pad_seq)
        lang_ids = torch.full((len(lens),), LANGUAGES.index(RUN), dtype=torch.long)
        with torch.no_grad():
            r = m(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), lang_ids=lang_ids,
                  output_hidden_states=True)
        h = r.hidden_states[-1]
        mk = torch.from_numpy(mask)[..., None].float()
        key = f"xmod_{preset}_{seed}_{scale}"
        out[key + "_ids"] = ids.astype(np.int32)
        out[key + "_mask"] = mask.astype(np.int8)
        out[key + "_mean"] = torch.nn.functional.normalize((h * mk).sum(1) / mk.sum(1).clamp(min=1e-9), p=2, dim=1).numpy()
        out[key + "_cls"] = torch.nn.functional.normalize(h[:, 0], p=2, dim=1).numpy()
        out[key + "_h_first"] = h[:, 0].numpy()
        out[key + "_h_last"] = np.stack([h[b, n - 1].numpy() for b, n in enumerate(lens)])
        out[key + "_logits"] = r.logits.numpy()
    return out


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    np.savez_compressed(os.path.join(HERE, "xmod.npz"), **xmod_goldens())
    print("xmod.npz", os.path.getsize(os.path.join(HERE, "xmod.npz")) // 1024, "KiB")
