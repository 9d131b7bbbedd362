"""Writes tests/golden/qwen3.npz from transformers 5.5's Qwen3Model, Qwen3ForSequenceClassification and
Qwen3ForCausalLM (eager attention, fp32) on the seeded weights of the ``tiny-qwen3`` shape, with a byte-level BPE
tokenizer built here (the Qwen specials, single ``yes`` / ``no`` tokens, and a post-processor that appends
<|endoftext|>, which is also the pad id, so the sequence-classification head must skip it).

    python tests/golden/make_golden_qwen3.py

``build()`` and ``save_snapshots()`` are shared with the tests, which save the same models as snapshots.  The zip
entries have fixed timestamps, so rerunning the script writes the same bytes.
"""
from __future__ import annotations

import io
import json
import os
import sys
import zipfile
from dataclasses import asdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from ragmeup_b200.tokenizer import build_byte_bpe  # noqa: E402
from ragmeup_b200.weights import (PRESETS, QWEN3_RERANK_INSTRUCTION, QWEN3_RERANK_PREFIX,  # noqa: E402
                                  QWEN3_RERANK_SUFFIX, Qwen3Config, synthetic_qwen3_weights)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "qwen3.npz")
WORDS = ["yes", "no", "query", "document", "passage", "search", "answer", "retrieve", "relevant", "web", "given",
         "the", "of", "and", "to", "in", "is", "that", "for", "on", "with", "as", "by", "at", "from", "data", "model"]
SEED, SCALE = 3, 2.0


def tokenizer():
    return build_byte_bpe(WORDS, append="<|endoftext|>")


def texts(n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    vocab = WORDS + ["GPU", "H100", "kernel", "Zürich", "naïve", "x=1", "42", "e.g.", "(a)", "don't"]
    return [" ".join(vocab[int(j)] for j in rng.integers(0, len(vocab), int(rng.integers(lo, hi + 1)))) for _ in range(n)]


def build():
    """(cfg, canonical weights with the sequence-classification head, lm_head [V, H], tokenizer) of the fixture"""
    tok = tokenizer()
    cfg = Qwen3Config(**asdict(PRESETS["tiny-qwen3"][0]))
    cfg.pad_token_id = tok.token_to_id("<|endoftext|>")
    w = synthetic_qwen3_weights(cfg, seed=SEED, with_head=True, scale=SCALE)
    rng = np.random.default_rng(SEED + 1)
    lm = (0.02 * SCALE * rng.standard_normal((cfg.vocab_size, cfg.hidden))).astype(np.float32)
    return cfg, w, lm, tok


def hf_config(cfg, attn="eager", **kw):
    import transformers
    return transformers.Qwen3Config(
        vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, intermediate_size=cfg.ffn, num_hidden_layers=cfg.layers,
        num_attention_heads=cfg.heads, num_key_value_heads=cfg.kv_heads, head_dim=cfg.head_dim,
        max_position_embeddings=cfg.max_pos, rms_norm_eps=cfg.ln_eps,
        rope_parameters={"rope_type": "default", "rope_theta": cfg.rope_theta}, tie_word_embeddings=False,
        pad_token_id=cfg.pad_token_id, attn_implementation=attn, **kw)


def hf_models(cfg, w, lm, attn="eager"):
    """the three transformers models on the fixture's weights: (Qwen3Model, Qwen3ForSequenceClassification,
    Qwen3ForCausalLM).  Eager attention takes its softmax in float32 whatever the model's dtype; "sdpa" keeps float64."""
    import transformers
    body = {k: torch.from_numpy(v) for k, v in w.items() if k != "head"}
    base = transformers.Qwen3Model(hf_config(cfg, attn)).eval()
    base.load_state_dict(body, strict=True)
    seq = transformers.Qwen3ForSequenceClassification(hf_config(cfg, attn, num_labels=1)).eval()
    seq.load_state_dict({**{"model." + k: v for k, v in body.items()}, "score.weight": torch.from_numpy(w["head"])},
                        strict=True)
    lmm = transformers.Qwen3ForCausalLM(hf_config(cfg, attn)).eval()
    lmm.load_state_dict({**{"model." + k: v for k, v in body.items()}, "lm_head.weight": torch.from_numpy(lm)}, strict=True)
    return base, seq, lmm


def save_snapshots(root, cfg, w, lm, tok, bf16: bool = False):
    """three snapshot directories under root: ``embedder`` (Qwen3Model with sentence-transformers' last-token Pooling
    and Normalize), ``seqcls`` and ``reranker`` (Qwen3ForCausalLM); bf16 saves the weights as bfloat16"""
    base, seq, lmm = hf_models(cfg, w, lm)
    out = {}
    for name, m in (("embedder", base), ("seqcls", seq), ("reranker", lmm)):
        d = os.path.join(root, name)
        if bf16:
            m = m.to(torch.bfloat16)
        m.save_pretrained(d, safe_serialization=True)
        tok.save(os.path.join(d, "tokenizer.json"))
        out[name] = d
    d = out["embedder"]
    with open(os.path.join(d, "modules.json"), "w") as f:
        json.dump([{"idx": 0, "name": "0", "path": "", "type": "sentence_transformers.models.Transformer"},
                   {"idx": 1, "name": "1", "path": "1_Pooling", "type": "sentence_transformers.models.Pooling"},
                   {"idx": 2, "name": "2", "path": "2_Normalize", "type": "sentence_transformers.models.Normalize"}], f)
    os.makedirs(os.path.join(d, "1_Pooling"), exist_ok=True)
    with open(os.path.join(d, "1_Pooling", "config.json"), "w") as f:
        json.dump({"word_embedding_dimension": cfg.hidden, "pooling_mode_cls_token": False,
                   "pooling_mode_mean_tokens": False, "pooling_mode_lasttoken": True}, f)
    with open(os.path.join(d, "sentence_bert_config.json"), "w") as f:
        json.dump({"max_seq_length": 1024, "do_lower_case": False}, f)
    return out


def _pack(seqs):
    cu = np.zeros(len(seqs) + 1, np.int32)
    np.cumsum([len(s) for s in seqs], out=cu[1:])
    return np.concatenate([np.asarray(s, np.int32) for s in seqs]), cu


def compute():
    from transformers import PreTrainedTokenizerFast
    cfg, w, lm, tok = build()
    base, seq, lmm = hf_models(cfg, w, lm)
    emb_seqs = [e.ids for e in tok.encode_batch(texts(6, 1, 120, 1) + texts(1, 700, 700, 2))]
    qs, ds = texts(3, 2, 8, 3), texts(4, 10, 200, 4)
    pairs = [(q, d) for q in qs for d in ds]
    cls_seqs = [e.ids for e in tok.encode_batch(pairs)]
    hf_tok = PreTrainedTokenizerFast(tokenizer_object=tok)
    from oracle.qwen3_ref import rerank_ids
    rr_seqs = rerank_ids(hf_tok, QWEN3_RERANK_PREFIX, QWEN3_RERANK_SUFFIX, QWEN3_RERANK_INSTRUCTION, pairs, 8192)
    yes, no = tok.token_to_id("yes"), tok.token_to_id("no")
    with torch.no_grad():
        emb = np.stack([torch.nn.functional.normalize(base(torch.tensor([s])).last_hidden_state[0, -1], dim=-1).numpy()
                        for s in emb_seqs])
        cls = np.stack([seq(torch.tensor([s])).logits[0].numpy() for s in cls_seqs])
        rr = []
        for s in rr_seqs:
            lg = lmm(torch.tensor([s])).logits[0, -1]
            rr.append(float(torch.stack([lg[no], lg[yes]]).log_softmax(0)[1].exp()))
    e_ids, e_cu = _pack(emb_seqs)
    c_ids, c_cu = _pack(cls_seqs)
    r_ids, r_cu = _pack(rr_seqs)
    return {"emb_ids": e_ids, "emb_cu": e_cu, "emb": emb.astype(np.float32), "cls_ids": c_ids, "cls_cu": c_cu,
            "cls_logits": cls.astype(np.float32), "rr_ids": r_ids, "rr_cu": r_cu, "rr_scores": np.asarray(rr, np.float32),
            "yes_no": np.asarray([yes, no], np.int32)}


def write(arrays, path=OUT):
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            b = io.BytesIO()
            np.save(b, arrays[k], allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", date_time=(2020, 1, 1, 0, 0, 0)), b.getvalue())
    with open(path, "wb") as f:
        f.write(buf.getvalue())


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    write(compute())
    print(OUT)
