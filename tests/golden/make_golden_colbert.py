"""Mint tests/golden/colbert.npz from ``transformers.BertModel`` (attn_implementation="eager", fp32) fed the seeded
synthetic ColBERT weights the tests rebuild with ``ragmeup_b200.weights.synthetic_colbert``, then
``torch.nn.Linear(bias=False)``, ``F.normalize`` and MaxSim.  The query batch carries its [MASK] padding as query rows
that are masked out of ``attention_mask``, as ColBERT runs it.  Only token ids, masks and outputs are stored.

Usage:  python tests/golden/make_golden_colbert.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from ragmeup_b200.weights import synthetic_colbert  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
MASK, PAD = 103, 0

# (preset, seed, scale, query lengths (real tokens; padded to query_maxlen with [MASK]), document lengths)
CASES = [("colbertv2.0", 0, 1.0, [3, 9, 32], [3, 17, 60]),
         ("tiny-colbert", 2, 4.0, [3, 16, 7], [3, 64, 30, 5])]


def hf_model(cfg, w):
    from transformers import BertConfig, BertModel
    hc = BertConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, num_hidden_layers=cfg.layers,
                    num_attention_heads=cfg.heads, intermediate_size=cfg.ffn, max_position_embeddings=cfg.max_pos,
                    type_vocab_size=cfg.type_vocab, layer_norm_eps=cfg.ln_eps, hidden_act="gelu",
                    attn_implementation="eager")
    m = BertModel(hc, add_pooling_layer=False).eval()
    missing, unexpected = m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()}, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return m


def batch(rng, lens, S, vocab, marker, pad_with):
    ids = np.full((len(lens), S), pad_with, np.int64)
    mask = np.zeros((len(lens), S), np.int64)
    for b, n in enumerate(lens):
        s = np.r_[101, marker, rng.integers(200, vocab, max(n - 3, 0)), 102][:n]
        ids[b, :n] = s
        mask[b, :n] = 1
    return ids, mask


def main():
    out = {}
    for preset, seed, scale, qlens, dlens in CASES:
        cfg, w, lin, spec = synthetic_colbert(preset, seed, scale)
        rng = np.random.default_rng(seed + 100)
        qi, qm = batch(rng, qlens, spec.query_maxlen, cfg.vocab_size, 1, MASK)
        di, dm = batch(rng, dlens, max(dlens), cfg.vocab_size, 2, PAD)
        m = hf_model(cfg, w)
        linear = torch.nn.Linear(cfg.hidden, spec.dim, bias=False)
        with torch.no_grad():
            linear.weight.copy_(torch.from_numpy(lin))
            Q = torch.nn.functional.normalize(linear(m(torch.from_numpy(qi), attention_mask=torch.from_numpy(qm))[0]),
                                              p=2, dim=2)
            D = torch.nn.functional.normalize(linear(m(torch.from_numpy(di), attention_mask=torch.from_numpy(dm))[0]),
                                              p=2, dim=2)
            scores = []
            for i in range(len(qlens)):
                s = D @ Q[i].T
                s[torch.from_numpy(dm) == 0] = -9999
                scores.append(s.max(1).values.sum(-1))
            scores = torch.stack(scores)                                                             # [nq, nd]
        key = f"colbert_{preset}_{seed}_{scale}"
        out.update({key + "_qids": qi.astype(np.int32), key + "_qmask": qm.astype(np.int8),
                    key + "_dids": di.astype(np.int32), key + "_dmask": dm.astype(np.int8),
                    key + "_Q": Q.numpy().astype(np.float32), key + "_D": D.numpy().astype(np.float32),
                    key + "_scores": scores.numpy().astype(np.float32)})
    np.savez_compressed(os.path.join(HERE, "colbert.npz"), **out)


if __name__ == "__main__":
    main()
