"""Oracle: X-MOD (transformers ``XmodModel``, ``XmodForSequenceClassification``) on the CPU, the float64 reference of
the whole encoder with its language adapters, and ColBERT on a SentencePiece vocabulary (colbert-xm).  TEST
INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

What X-MOD computes that XLM-R does not (transformers ``models/xmod/modeling_xmod.py``, ``XmodOutput.lang_adapter`` with
the flags of facebook/xmod-base: pre_norm false, adapter_layer_norm false, adapter_reuse_layer_norm true,
ln_before_adapter true): with LN the layer's ``output.LayerNorm`` and y = W2 ffn + b2 + x1, a layer ends

    h = LN(y);  out = LN(D2 gelu(D1 h + d1) + d2 + h)

with the adapter (``output.adapter_modules.<language>.dense1`` / ``dense2``) of the sequence's language.  Embeddings,
positions, attention and the classification head are XLM-R's (``xlmr_ref``).

ColBERT on a SentencePiece vocabulary restates ``colbert_ref``'s rules with the tokenizer's own specials: <s> / </s>,
<pad> (id 1) for padding, <mask> for the query padding and for any literal pad id in a query, and a marker token the
vocabulary lacks as <unk> (``convert_tokens_to_ids``) [3P-recall: colbert-ai 0.2.x, not installed here].  Weight dicts
use the canonical names of ``ragmeup_b200.weights.weight_names``.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Sequence, Tuple

import numpy as np
import torch
from tokenizers import Tokenizer

from . import bert_ref, colbert_ref
from . import encoder_kernels_ref as ekr
from . import mpnet_ref, xlmr_ref

# rmu_encoder_create uploads these as split planes: the six of every layer and the adapter's two
GEMM_WEIGHTS = ekr.GEMM_WEIGHTS + ("dense1.weight", "dense2.weight")


@dataclass
class XmodCfg(xlmr_ref.XLMRCfg):
    adapter_dim: int = 384
    languages: Tuple[str, ...] = ("en_XX", "de_DE", "fr_XX")
    language: str = "en_XX"


def adapter(layer: int, language: str) -> Tuple[str, str, str, str]:
    """canonical names of one adapter: dense1.weight, dense1.bias, dense2.weight, dense2.bias"""
    p = f"encoder.layer.{layer}.output.adapter_modules.{language}."
    return p + "dense1.weight", p + "dense1.bias", p + "dense2.weight", p + "dense2.bias"


def xmod_encoder_forward(w: Dict[str, object], cfg, input_ids: torch.Tensor, attention_mask: torch.Tensor,
                         language: str = None, matmul=None, device=None) -> torch.Tensor:
    """[B, S] ids / mask -> last hidden state [B, S, H], fp32, padded with id 1: ``xlmr_ref.xlmr_encoder_forward`` with
    the adapter of ``language`` (default ``cfg.language``) in every layer."""
    mm = matmul or (lambda x, W: x @ W.t())
    dev = device or "cpu"
    lang = language or cfg.language
    tw = lambda a: bert_ref._t(a, dev)  # noqa: E731
    input_ids, attention_mask = input_ids.to(dev), attention_mask.to(dev)
    B, S = input_ids.shape
    H, nh = cfg.hidden, cfg.heads
    dh = H // nh
    x = (tw(w["embeddings.word_embeddings.weight"])[input_ids] + tw(w["embeddings.token_type_embeddings.weight"])[0]) + \
        tw(w["embeddings.position_embeddings.weight"])[xlmr_ref.position_ids(input_ids)]
    x = bert_ref._layer_norm(x, tw(w["embeddings.LayerNorm.weight"]), tw(w["embeddings.LayerNorm.bias"]), cfg.ln_eps)
    add_mask = (1.0 - attention_mask.to(torch.float32))[:, None, None, :] * torch.finfo(torch.float32).min
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}."
        q = mm(x, tw(w[p + "attention.self.query.weight"])) + tw(w[p + "attention.self.query.bias"])
        k = mm(x, tw(w[p + "attention.self.key.weight"])) + tw(w[p + "attention.self.key.bias"])
        v = mm(x, tw(w[p + "attention.self.value.weight"])) + tw(w[p + "attention.self.value.bias"])
        q = q.view(B, S, nh, dh).transpose(1, 2)
        k = k.view(B, S, nh, dh).transpose(1, 2)
        v = v.view(B, S, nh, dh).transpose(1, 2)
        att = torch.softmax(torch.matmul(q, k.transpose(2, 3)) * (dh ** -0.5) + add_mask, dim=-1)
        ctx = torch.matmul(att, v).transpose(1, 2).reshape(B, S, H)
        o = mm(ctx, tw(w[p + "attention.output.dense.weight"])) + tw(w[p + "attention.output.dense.bias"])
        x = bert_ref._layer_norm(o + x, tw(w[p + "attention.output.LayerNorm.weight"]),
                                 tw(w[p + "attention.output.LayerNorm.bias"]), cfg.ln_eps)
        f = bert_ref._gelu_erf(mm(x, tw(w[p + "intermediate.dense.weight"])) + tw(w[p + "intermediate.dense.bias"]))
        o = mm(f, tw(w[p + "output.dense.weight"])) + tw(w[p + "output.dense.bias"])
        g, b = tw(w[p + "output.LayerNorm.weight"]), tw(w[p + "output.LayerNorm.bias"])
        h = bert_ref._layer_norm(o + x, g, b, cfg.ln_eps)
        d1w, d1b, d2w, d2b = (tw(w[n]) for n in adapter(l, lang))
        z = (mm(bert_ref._gelu_erf(mm(h, d1w) + d1b), d2w) + d2b) + h
        x = bert_ref._layer_norm(z, g, b, cfg.ln_eps)
    return x


classifier_head = xlmr_ref.classifier_head


# ------------------------------------------------------------------------------------------ float64 whole encoder

def xmod_stack_ref(w, cfg, ids, cu, weights: str = "fp32", device=None, nkeys=None, language: str = None) -> dict:
    """The whole X-MOD encoder in float64 on the ragged batch (ids [T], cu [B + 1]), composed of the kernel references
    in the order the device runs them: XLM-R's position rule and type row 0, attention (keys of sequence b limited to
    its first nkeys[b] rows when given, ColBERT's query padding), and after the FFN-out GEMM the adapter: LN2 -> D1 with
    erf-GELU -> D2 + bias + h -> LN2.  weights "fp32" as given, "split" as hi + lo of the split planes (the adapter's
    dense weights included).  Returns {"hidden": [T, H], "mean" / "cls" / "mean_norm" / "cls_norm": [B, H], and
    "logits" [B, num_labels] when w holds the head}, float64 on ``device``."""
    if weights not in ("fp32", "split"):
        raise ValueError(weights)
    dev = torch.device(device or "cpu")
    lang = language or cfg.language
    W = lambda name: (ekr.split_weight(w[name]) if weights == "split" else ekr._f64(w[name])).to(dev)  # noqa: E731
    V = lambda name: ekr._f64(w[name]).to(dev)                                                            # noqa: E731
    cu_l = [int(c) for c in cu]
    nk = [c1 - c0 for c0, c1 in zip(cu_l[:-1], cu_l[1:])] if nkeys is None else [int(n) for n in nkeys]
    H, heads, eps = cfg.hidden, cfg.heads, float(cfg.ln_eps)
    x = mpnet_ref.embed_ln_pos_ref(ekr._long(ids, dev), None, ekr._long(cu_l, dev), V("embeddings.word_embeddings.weight"),
                                   V("embeddings.position_embeddings.weight"),
                                   V("embeddings.token_type_embeddings.weight"), V("embeddings.LayerNorm.weight"),
                                   V("embeddings.LayerNorm.bias"), eps)[0]
    qs = math.log2(math.e) / math.sqrt(H // heads)
    z = torch.zeros_like
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}."
        wqkv = torch.cat([W(p + "attention.self." + n + ".weight") for n in ("query", "key", "value")])
        bqkv = torch.cat([V(p + "attention.self." + n + ".bias") for n in ("query", "key", "value")])
        qkv = ekr.gemm_ref(ekr.GEMM_BIAS_F32, x, z(x), wqkv, z(wqkv), bqkv)[0]
        qkv[:, :H] *= qs
        ctx = colbert_ref.attention_keys_ref(qkv, z(qkv), cu_l, nk, heads)[0]
        wo = W(p + "attention.output.dense.weight")
        o = ekr.gemm_ref(ekr.GEMM_BIAS_RESID_F32, ctx, z(ctx), wo, z(wo), V(p + "attention.output.dense.bias"), x, z(x))[0]
        x1 = ekr.layernorm_ref(o, V(p + "attention.output.LayerNorm.weight"), V(p + "attention.output.LayerNorm.bias"),
                               eps)[0]
        w1 = W(p + "intermediate.dense.weight")
        f = ekr.gemm_ref(ekr.GEMM_BIAS_GELU_SPLIT, x1, z(x1), w1, z(w1), V(p + "intermediate.dense.bias"))[0]
        w2 = W(p + "output.dense.weight")
        y = ekr.gemm_ref(ekr.GEMM_BIAS_RESID_F32, f, z(f), w2, z(w2), V(p + "output.dense.bias"), x1, z(x1))[0]
        g, b = V(p + "output.LayerNorm.weight"), V(p + "output.LayerNorm.bias")
        h = ekr.layernorm_ref(y, g, b, eps)[0]
        n1w, n1b, n2w, n2b = adapter(l, lang)
        d1, d2 = W(n1w), W(n2w)
        a = ekr.gemm_ref(ekr.GEMM_BIAS_GELU_SPLIT, h, z(h), d1, z(d1), V(n1b))[0]
        zz = ekr.gemm_ref(ekr.GEMM_BIAS_RESID_F32, a, z(a), d2, z(d2), V(n2b), h, z(h))[0]
        x = ekr.layernorm_ref(zz, g, b, eps)[0]
    out = {"hidden": x}
    for mode, name in ((0, "mean"), (1, "cls")):
        out[name] = ekr.pool_ref(x, z(x), cu_l, mode, False)[0]
        out[name + "_norm"] = ekr.pool_ref(x, z(x), cu_l, mode, True)[0]
    if "pooler.dense.weight" in w:
        out["logits"] = ekr.cls_head_ref(x, z(x), cu_l, V("pooler.dense.weight"), V("pooler.dense.bias"),
                                         V("classifier.weight"), V("classifier.bias"))[0]
    return out


def colbert_stack_ref(w, cfg, linear, ids, cu, nkeys=None, keep=None, weights: str = "split", device=None) -> Dict:
    """``xmod_stack_ref`` with the key limit, then ``linear`` (split planes with weights = "split") and the
    normalisation; tokens with keep 0 get zero vectors.  Returns {"hidden", "vectors"} float64."""
    dev = torch.device(device or "cpu")
    x = xmod_stack_ref(w, cfg, ids, cu, weights, device=dev, nkeys=nkeys)["hidden"]
    lin = (ekr.split_weight(linear) if weights == "split" else ekr._f64(linear)).to(dev)
    proj = x @ lin.T
    vec = proj / proj.norm(dim=1, keepdim=True).clamp(min=1e-12)
    if keep is not None:
        vec = vec * torch.as_tensor(np.asarray(keep) != 0, device=dev)[:, None]
    return {"hidden": x, "vectors": vec}


# --------------------------------------------------------------------------- ColBERT on a SentencePiece vocabulary

def specials(tok: Tokenizer, spec) -> Dict[str, int]:
    """<pad>, <mask> and the markers (a marker the vocabulary lacks is <unk>)"""
    unk = tok.token_to_id("<unk>")
    q, d = tok.token_to_id(spec.query_token), tok.token_to_id(spec.doc_token)
    return {"pad": tok.token_to_id("<pad>"), "mask": tok.token_to_id("<mask>"), "q": unk if q is None else q,
            "d": unk if d is None else d}


def tokenize_queries(tok: Tokenizer, spec, texts: Sequence[str]) -> Tuple[torch.Tensor, torch.Tensor]:
    """-> (ids [n, query_maxlen], attention_mask [n, query_maxlen]) int64: padding="max_length" with <pad>, position
    1 = the query marker, every pad id -> <mask>"""
    t = colbert_ref._copy(tok)
    s = specials(t, spec)
    t.enable_truncation(max_length=spec.query_maxlen)
    t.enable_padding(pad_id=s["pad"], pad_token="<pad>", length=spec.query_maxlen)
    enc = t.encode_batch([". " + x for x in texts])
    ids = torch.tensor([e.ids for e in enc], dtype=torch.long)
    am = torch.tensor([e.attention_mask for e in enc], dtype=torch.long)
    ids[:, 1] = s["q"]
    ids[ids == s["pad"]] = s["mask"]
    return ids, am


def tokenize_docs(tok: Tokenizer, spec, texts: Sequence[str]) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """-> (ids [n, S], attention_mask [n, S], score mask [n, S]): the score mask drops the skiplist and the pad id"""
    t = colbert_ref._copy(tok)
    s = specials(t, spec)
    t.enable_truncation(max_length=spec.doc_maxlen, strategy="longest_first")
    t.enable_padding(pad_id=s["pad"], pad_token="<pad>")
    enc = t.encode_batch([". " + x for x in texts])
    ids = torch.tensor([e.ids for e in enc], dtype=torch.long)
    am = torch.tensor([e.attention_mask for e in enc], dtype=torch.long)
    ids[:, 1] = s["d"]
    skip = set(colbert_ref.skiplist(t)) if spec.mask_punctuation else set()
    keep = torch.tensor([[(x not in skip) and (x != s["pad"]) for x in row] for row in ids.tolist()], dtype=torch.bool)
    return ids, am, keep


def vectors(w, cfg, linear, ids: torch.Tensor, attention_mask: torch.Tensor, device=None) -> torch.Tensor:
    """fp32 forward -> normalize(linear(h)) [n, S, dim]"""
    with torch.no_grad():
        h = xmod_encoder_forward(w, cfg, ids, attention_mask, device=device)
        return torch.nn.functional.normalize(h @ bert_ref._t(linear, h.device).T, p=2, dim=2)


def score_pairs(w, cfg, linear, spec, tok: Tokenizer, pairs: Sequence[Tuple[str, str]], device=None) -> np.ndarray:
    """HuggingFaceCrossEncoder.score on colbert-xm: ``colbert_ref.score_pairs`` with the rules above"""
    if len(pairs) == 0:
        raise IndexError("score_pairs: empty input")
    queries = list(dict.fromkeys(p[0] for p in pairs))
    docs = list(dict.fromkeys(p[1] for p in pairs))
    qi, am = tokenize_queries(tok, spec, queries)
    Q = vectors(w, cfg, linear, qi, am, device)
    D_all = {}
    for s in range(0, len(docs), 32):
        chunk = docs[s:s + 32]
        di, dam, keep = tokenize_docs(tok, spec, chunk)
        D = vectors(w, cfg, linear, di, dam, device)
        for j, d in enumerate(chunk):
            D_all[d] = (D[j:j + 1], keep[j:j + 1])
    qpos = {q: i for i, q in enumerate(queries)}
    out = np.empty(len(pairs), np.float32)
    for n, (q, d) in enumerate(pairs):
        D, keep = D_all[d]
        out[n] = float(colbert_ref.colbert_score(Q[qpos[q]], D, keep)[0])
    return out
