"""Mint tests/golden/modernbert.npz from ``transformers.ModernBertForSequenceClassification`` (attn_implementation="eager",
fp32) fed the seeded synthetic weights the tests rebuild with ``ragmeup_b200.weights.synthetic_bert_weights``; only
token ids, masks and outputs are stored.  Both tiny presets (half-window 64, and 16 so short sequences cross many
window blocks), CLS and mean pooling, lengths across the window (65, 66, 129), the 160-row attention CTA edge (161)
and past 600 tokens.  Each sequence runs alone (batch of one, no padding).  Separate from the other generators, so
their golden files are not rewritten.

Usage:  python tests/golden/make_golden_modernbert.py
"""
import io
import os
import sys
import zipfile
from dataclasses import asdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from ragmeup_b200.weights import PRESETS, ModernBertConfig, synthetic_bert_weights  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CLS_ID, SEP_ID, PAD_ID = 101, 102, 0      # the synthetic WordPiece vocabulary's, inside every tiny vocabulary

# (preset, seed, scale, pooling, lengths)
CASES = [("tiny-modernbert", 0, 1.0, "cls", [1, 65, 66, 129, 161, 640]),
         ("tiny-modernbert", 3, 4.0, "mean", [2, 65, 129, 161, 700]),
         ("tiny-modernbert-window", 1, 1.0, "mean", [17, 65, 66, 161, 640]),
         ("tiny-modernbert-window", 2, 4.0, "cls", [33, 66, 129, 161, 600])]


def case_key(preset, seed, scale, pooling):
    return f"modernbert_{preset}_{seed}_{scale}_{pooling}"


def case_config(preset, pooling) -> ModernBertConfig:
    cfg = ModernBertConfig(**asdict(PRESETS[preset][0]))
    cfg.classifier_pooling = pooling
    return cfg


def hf_model(cfg: ModernBertConfig, w):
    """ModernBertForSequenceClassification with cfg's shape, layer types, window and pooling, holding w (no biases,
    no LayerNorm shifts: transformers' defaults, which synthetic_bert_weights follows with zeros)"""
    from transformers import ModernBertConfig as HFConfig, ModernBertForSequenceClassification
    halves = {x for x in cfg.layer_windows if x}
    assert len(halves) <= 1, "transformers has one window size per model"
    hc = HFConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, num_hidden_layers=cfg.layers,
                  num_attention_heads=cfg.heads, intermediate_size=cfg.ffn, max_position_embeddings=cfg.max_pos,
                  norm_eps=cfg.ln_eps, layer_types=["full_attention" if x == 0 else "sliding_attention"
                                                    for x in cfg.layer_windows],
                  local_attention=2 * (halves.pop() if halves else 64),
                  rope_parameters={"full_attention": {"rope_type": "default", "rope_theta": cfg.global_theta},
                                   "sliding_attention": {"rope_type": "default", "rope_theta": cfg.local_theta}},
                  classifier_pooling=cfg.classifier_pooling, num_labels=cfg.num_labels, pad_token_id=PAD_ID,
                  bos_token_id=CLS_ID, eos_token_id=SEP_ID, cls_token_id=CLS_ID, sep_token_id=SEP_ID,
                  attn_implementation="eager")
    m = ModernBertForSequenceClassification(hc).eval()
    sd = {}
    for k, v in w.items():
        if k.startswith("layers.0.attn_norm.") or (k.endswith(".bias") and not k.startswith("classifier.")):
            assert not np.any(v != (1.0 if k.endswith("weight") else 0.0)), k   # placeholders and zero biases only
            continue
        sd[k if k.startswith(("head.", "classifier.")) else "model." + k] = torch.from_numpy(v)
    m.load_state_dict(sd, strict=True)
    return m


def batch(rng, cfg, lens):
    """[CLS] ... [SEP] sequences, padded with [PAD] into [B, max(lens)] (the padding is not run)"""
    ids = np.full((len(lens), max(lens)), PAD_ID, dtype=np.int32)
    mask = np.zeros(ids.shape, dtype=np.int8)
    for b, n in enumerate(lens):
        ids[b, :n] = rng.integers(103, cfg.vocab_size, n)
        ids[b, 0] = CLS_ID
        if n > 1:
            ids[b, n - 1] = SEP_ID
        mask[b, :n] = 1
    return ids, mask


def modernbert_goldens():
    rng = np.random.default_rng(2026)
    out = {}
    for preset, seed, scale, pooling, lens in CASES:
        cfg = case_config(preset, pooling)
        w = synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale)
        m = hf_model(cfg, w)
        ids, mask = batch(rng, cfg, lens)
        h_first, h_last, h_mean, logits = [], [], [], []
        with torch.no_grad():
            for b, n in enumerate(lens):
                r = m(input_ids=torch.from_numpy(ids[b:b + 1, :n].astype(np.int64)), output_hidden_states=True)
                h = r.hidden_states[-1][0]
                h_first.append(h[0].numpy())
                h_last.append(h[n - 1].numpy())
                h_mean.append(h.mean(0).numpy())
                logits.append(r.logits[0].numpy())
        key = case_key(preset, seed, scale, pooling)
        out[key + "_ids"] = ids
        out[key + "_mask"] = mask
        out[key + "_h_first"] = np.stack(h_first)
        out[key + "_h_last"] = np.stack(h_last)
        out[key + "_h_mean"] = np.stack(h_mean)
        out[key + "_logits"] = np.stack(logits)
    return out


def save_reproducibly(path, arrays):
    """np.savez_compressed with fixed zip entry times, so a rerun writes the same bytes"""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.save(buf, np.ascontiguousarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    path = os.path.join(HERE, "modernbert.npz")
    save_reproducibly(path, modernbert_goldens())
    print("modernbert.npz", os.path.getsize(path) // 1024, "KiB")
