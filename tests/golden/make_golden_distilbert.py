"""Mint tests/golden/distilbert.npz from transformers' ``DistilBertModel`` and ``DistilBertForSequenceClassification``
(eager attention, float64) fed the seeded synthetic weights the tests rebuild with
``ragmeup_b200.weights.synthetic_bert_weights`` / ``synthetic_dense_weights``, and from ``oracle.dense_ref`` for two
Dense chains: "tanh" (128 -> 300 tanh with bias, 300 -> 160 identity without bias: widening, then narrowing) and
"identity" (128 -> 96 identity without bias).  Only ids and outputs are stored.

Usage:  python tests/golden/make_golden_distilbert.py
"""
import os
import sys
from dataclasses import asdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import dense_ref  # noqa: E402
from ragmeup_b200.weights import (PRESETS, DistilBertConfig, dense_layers, synthetic_bert_weights,  # noqa: E402
                                  synthetic_dense_weights)

HERE = os.path.dirname(os.path.abspath(__file__))
PRESET, SEED, SCALE = "tiny-distilbert", 5, 2.0
CHAINS = {"tanh": ((300, True, "tanh"), (160, False, "identity")), "identity": ((96, False, "identity"),)}
LENS = [1, 9, 16, 64, 2, 33, 40]


def config() -> DistilBertConfig:
    return DistilBertConfig(**{**asdict(PRESETS[PRESET][0]), "num_labels": 3})


def weights(cfg: DistilBertConfig):
    """(encoder + head weights, {chain: Dense weights}) in the canonical names"""
    w = synthetic_bert_weights(cfg, seed=SEED, with_head=True, scale=SCALE)
    return w, {name: synthetic_dense_weights(cfg.hidden, layers, seed=SEED + i, scale=SCALE * 3)
               for i, (name, layers) in enumerate(CHAINS.items())}


def hf_state_dict(w, prefix=""):
    """canonical (BERT) names -> DistilBERT's (``prefix`` = "distilbert." for the classification model's encoder)"""
    ren = (("encoder.layer.", "transformer.layer."), ("attention.self.query.", "attention.q_lin."),
           ("attention.self.key.", "attention.k_lin."), ("attention.self.value.", "attention.v_lin."),
           ("attention.output.dense.", "attention.out_lin."), ("attention.output.LayerNorm.", "sa_layer_norm."),
           ("intermediate.dense.", "ffn.lin1."), ("output.dense.", "ffn.lin2."), ("output.LayerNorm.", "output_layer_norm."))
    sd = {}
    for k, v in w.items():
        if k == "embeddings.token_type_embeddings.weight" or k.startswith("dense."):
            continue
        if k.startswith("pooler.dense."):
            sd["pre_classifier." + k[13:]] = torch.from_numpy(v)
            continue
        if k.startswith("classifier."):
            sd[k] = torch.from_numpy(v)
            continue
        for a, b in ren:
            k = k.replace(a, b)
        sd[prefix + k] = torch.from_numpy(v)
    return sd


def hf_config(cfg: DistilBertConfig, sinusoidal: bool = False):
    from transformers import DistilBertConfig as HC
    return HC(vocab_size=cfg.vocab_size, dim=cfg.hidden, n_layers=cfg.layers, n_heads=cfg.heads, hidden_dim=cfg.ffn,
              max_position_embeddings=cfg.max_pos, num_labels=cfg.num_labels, dropout=0.0, attention_dropout=0.0,
              seq_classif_dropout=0.0, sinusoidal_pos_embds=sinusoidal, attn_implementation="eager")


def hf_models(cfg: DistilBertConfig, w):
    from transformers import DistilBertForSequenceClassification, DistilBertModel
    base = DistilBertModel(hf_config(cfg)).eval()
    r = base.load_state_dict({k: v for k, v in hf_state_dict(w).items()
                              if not k.startswith(("pre_classifier.", "classifier."))}, strict=False)
    assert not r.missing_keys and not r.unexpected_keys, r
    head = DistilBertForSequenceClassification(hf_config(cfg)).eval()
    r = head.load_state_dict(hf_state_dict(w, "distilbert."), strict=False)
    assert not r.missing_keys and not r.unexpected_keys, r
    return base.double(), head.double()


def batch(cfg: DistilBertConfig):
    rng = np.random.default_rng(11)
    seqs = [np.r_[101, rng.integers(5, cfg.vocab_size, max(n - 2, 0)), 102][:n] for n in LENS]
    ids = np.concatenate(seqs).astype(np.int32)
    return ids, np.r_[0, np.cumsum(LENS)].astype(np.int32)


def write_snapshot(path: str, cfg: DistilBertConfig, head: bool = False, dense=((200, True, "tanh"),),
                   pooling: str = "mean", normalize: bool = False, dense_format: str = "safetensors", seed: int = 0,
                   sinusoidal: bool = False):
    """a sentence-transformers / HF snapshot of a randomly initialised transformers DistilBERT (torch seed ``seed``):
    config.json and model.safetensors by ``save_pretrained``, vocab.txt of the synthetic WordPiece vocabulary, and
    without ``head`` modules.json with Pooling, one ``<i+2>_Dense`` directory per entry of ``dense`` ((out_features,
    bias, "tanh" | "identity"), weights in ``dense_format`` "safetensors" or "bin") and Normalize when asked.  Returns
    (the float64 transformers model, {Dense dir: (weight, bias or None, act code)})."""
    import json
    from transformers import DistilBertForSequenceClassification, DistilBertModel
    from ragmeup_b200.tokenizer import synthetic_vocab
    torch.manual_seed(seed)
    model = (DistilBertForSequenceClassification if head else DistilBertModel)(hf_config(cfg, sinusoidal)).eval()
    model.save_pretrained(path, safe_serialization=True)
    vocab = synthetic_vocab(cfg.vocab_size)
    with open(os.path.join(path, "vocab.txt"), "w", encoding="utf-8") as f:
        f.write("\n".join(sorted(vocab, key=vocab.get)) + "\n")
    layers = {}
    if not head:
        mods = [{"path": "", "type": "sentence_transformers.models.Transformer"},
                {"path": "1_Pooling", "type": "sentence_transformers.models.Pooling"}]
        os.makedirs(os.path.join(path, "1_Pooling"), exist_ok=True)
        with open(os.path.join(path, "1_Pooling", "config.json"), "w") as f:
            json.dump({"pooling_mode_cls_token": pooling == "cls", "pooling_mode_mean_tokens": pooling == "mean"}, f)
        d_in = cfg.hidden
        for i, (d_out, bias, act) in enumerate(dense):
            mdir = f"{i + 2}_Dense"
            os.makedirs(os.path.join(path, mdir), exist_ok=True)
            lin = torch.nn.Linear(d_in, d_out, bias=bias)
            sd = {k: v.detach().contiguous() for k, v in lin.state_dict().items()}
            sd = {"linear." + k: v for k, v in sd.items()}
            if dense_format == "bin":
                torch.save(sd, os.path.join(path, mdir, "pytorch_model.bin"))
            else:
                from safetensors.torch import save_file
                save_file(sd, os.path.join(path, mdir, "model.safetensors"))
            cls = {"tanh": "torch.nn.modules.activation.Tanh", "identity": "torch.nn.modules.linear.Identity"}[act]
            with open(os.path.join(path, mdir, "config.json"), "w") as f:
                json.dump({"in_features": d_in, "out_features": d_out, "bias": bias, "activation_function": cls}, f)
            mods.append({"path": mdir, "type": "sentence_transformers.models.Dense"})
            layers[mdir] = (sd["linear.weight"].numpy(), sd["linear.bias"].numpy() if bias else None,
                            {"identity": 0, "tanh": 1}[act])
            d_in = d_out
        if normalize:
            mods.append({"path": f"{len(dense) + 2}_Normalize", "type": "sentence_transformers.models.Normalize"})
        with open(os.path.join(path, "modules.json"), "w") as f:
            json.dump(mods, f)
    return model.double(), layers


def make() -> dict:
    cfg = config()
    w, chains = weights(cfg)
    base, head = hf_models(cfg, w)
    ids, cu = batch(cfg)
    B, S = len(LENS), max(LENS)
    I = torch.zeros((B, S), dtype=torch.int64)
    M = torch.zeros((B, S), dtype=torch.int64)
    for b, n in enumerate(LENS):
        I[b, :n] = torch.from_numpy(ids[cu[b]:cu[b + 1]].astype(np.int64))
        M[b, :n] = 1
    with torch.no_grad():
        h = base(input_ids=I, attention_mask=M).last_hidden_state
        logits = head(input_ids=I, attention_mask=M).logits
    m = M[..., None].double()
    pooled = {"mean": (h * m).sum(1) / m.sum(1), "cls": h[:, 0]}
    out = {"ids": ids, "cu": cu, "seed": np.array(SEED), "scale": np.array(SCALE), "logits": logits.numpy()}
    for mode, p in pooled.items():
        out[f"pooled_{mode}"] = p.numpy()
        for name, dw in chains.items():
            for norm in (False, True):
                y = dense_ref.dense_chain_ref(p, dense_layers(dw), norm)
                out[f"{name}_{mode}{'_norm' if norm else ''}"] = y.numpy()
    return out


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "distilbert.npz"), **make())
    print("wrote", os.path.join(HERE, "distilbert.npz"))
