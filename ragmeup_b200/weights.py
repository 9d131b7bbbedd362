"""BERT-family model description + weight sources for the GPU encoder.

The reference names its models by HuggingFace id (``embedding_model`` /
``rerank_model`` in ``server/.env.template:3,43``; constructed at
``server/RAGHelper_local.py:114-117`` and ``server/RAGHelper.py:484``).  This
module resolves such a name to (config, weight dict, pooling rule) from

* a local HuggingFace / sentence-transformers snapshot directory
  (``config.json`` + ``model.safetensors`` [+ ``modules.json``,
  ``1_Pooling/config.json``, ``sentence_bert_config.json``]); or
* ``synthetic:<preset>[:seed]`` — seeded random-init weights of the named
  architecture.  There is no network in the build/bench image, so the
  benchmarks and parity tests use these (BASELINE.json configs only fix the
  *shapes*).

Weight dict keys are HuggingFace ``BertModel`` names without the ``bert.``
prefix; values are contiguous float32 numpy arrays.
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass, asdict
from typing import ClassVar, Dict, Optional, Tuple

import numpy as np


@dataclass
class BertConfig:
    vocab_size: int = 30522
    hidden: int = 384
    layers: int = 6
    heads: int = 12
    ffn: int = 1536
    max_pos: int = 512
    type_vocab: int = 2
    ln_eps: float = 1e-12
    num_labels: int = 1
    # BERT: positions 0..S-1, no relative bias, no language adapter (class constants, so asdict() of a BERT config keeps
    # its nine fields)
    position_mode: ClassVar[int] = 0
    rel_buckets: ClassVar[int] = 0
    adapter_dim: ClassVar[int] = 0
    # no disentangled attention, BERT's tanh pooler
    position_buckets: ClassVar[int] = 0
    max_relative_positions: ClassVar[int] = 0
    head_act: ClassVar[int] = 0

    @property
    def head_dim(self) -> int:
        return self.hidden // self.heads

    @property
    def position_offset(self) -> int:
        """first position row a token can take: a sequence may hold max_pos - position_offset tokens"""
        return 2 if self.position_mode == 1 else 0

    @staticmethod
    def from_hf(d: dict) -> "BertConfig":
        if d.get("hidden_act", "gelu") != "gelu":
            raise ValueError(f"only erf-GELU BERT encoders are supported, got {d.get('hidden_act')}")
        if d.get("position_embedding_type", "absolute") != "absolute":
            raise ValueError("only absolute position embeddings are supported")
        return BertConfig(
            vocab_size=d["vocab_size"], hidden=d["hidden_size"], layers=d["num_hidden_layers"],
            heads=d["num_attention_heads"], ffn=d["intermediate_size"],
            max_pos=d["max_position_embeddings"], type_vocab=d.get("type_vocab_size", 2),
            ln_eps=d.get("layer_norm_eps", 1e-12),
            num_labels=len(d["id2label"]) if "id2label" in d else d.get("num_labels", 1))


@dataclass
class MPNetConfig(BertConfig):
    """MPNet (transformers ``MPNetModel``): BERT's post-LN encoder with RoBERTa-style positions (padding index 1:
    positions start at 2, a token of id 1 takes position 1) and a relative position bias [32, heads] shared by every
    layer.  It has no token-type table; the encoder gets a zero [1, H] one, and (w + 0) + p == w + p exactly."""
    vocab_size: int = 30527
    max_pos: int = 514
    type_vocab: int = 1
    ln_eps: float = 1e-5
    position_mode: int = 1
    rel_buckets: int = 32

    @staticmethod
    def from_hf(d: dict) -> "MPNetConfig":
        if d.get("hidden_act", "gelu") != "gelu":
            raise ValueError(f"only erf-GELU MPNet encoders are supported, got {d.get('hidden_act')}")
        nb = int(d.get("relative_attention_num_buckets", 32))
        if nb < 32:
            raise ValueError(f"MPNet with relative_attention_num_buckets = {nb} is not supported: transformers' MPNet "
                             f"always looks up 32 buckets")
        return MPNetConfig(vocab_size=d["vocab_size"], hidden=d["hidden_size"], layers=d["num_hidden_layers"],
                           heads=d["num_attention_heads"], ffn=d["intermediate_size"],
                           max_pos=d["max_position_embeddings"], ln_eps=d.get("layer_norm_eps", 1e-12))


@dataclass
class XLMRConfig(BertConfig):
    """XLM-RoBERTa and RoBERTa (transformers ``XLMRobertaModel`` / ``RobertaModel``): BERT's post-LN encoder with
    MPNet's padding-offset positions (padding index 1) and no relative bias.  The [1, H] token-type table is a trained
    row, added to every token (the tokenizers return no token types).  The classification head
    (``RobertaClassificationHead``: dense, tanh, out_proj on token 0) is BERT's pooler + classifier."""
    vocab_size: int = 250002
    max_pos: int = 514
    type_vocab: int = 1
    ln_eps: float = 1e-5
    position_mode: int = 1
    rel_buckets: int = 0

    @staticmethod
    def from_hf(d: dict) -> "XLMRConfig":
        kind = d.get("model_type", "xlm-roberta")
        if int(d.get("pad_token_id", 1)) != 1:
            raise ValueError(f"{kind} with pad_token_id = {d['pad_token_id']} is not supported: the encoder's position "
                             f"rule has the padding index fixed at 1")
        if d.get("position_embedding_type", "absolute") != "absolute":
            raise ValueError(f"{kind}: only absolute position embeddings are supported, got "
                             f"{d['position_embedding_type']!r}")
        if d.get("hidden_act", "gelu") != "gelu":
            raise ValueError(f"only erf-GELU {kind} encoders are supported, got {d.get('hidden_act')}")
        return XLMRConfig(vocab_size=d["vocab_size"], hidden=d["hidden_size"], layers=d["num_hidden_layers"],
                          heads=d["num_attention_heads"], ffn=d["intermediate_size"],
                          max_pos=d["max_position_embeddings"], type_vocab=d.get("type_vocab_size", 1),
                          ln_eps=d.get("layer_norm_eps", 1e-5),
                          num_labels=len(d["id2label"]) if "id2label" in d else d.get("num_labels", 1))


@dataclass
class DistilBertConfig(BertConfig):
    """DistilBERT (transformers ``DistilBertModel`` / ``DistilBertForSequenceClassification``; distiluse-base-multilingual-
    cased-v2): BERT's post-LN encoder with erf-GELU, LayerNorm eps 1e-12, learned positions and BERT's attention scaling,
    under other tensor names (``distilbert_to_canonical``) and without token types.  The encoder gets a zero [1, H]
    token-type table, so no type id can select a non-zero row: (w + 0) + p == w + p exactly.  It runs BERT's forward as
    it is; only the head differs: ``classifier(relu(pre_classifier(h_CLS)))`` (``head_act`` RMU_HEAD_RELU)."""
    vocab_size: int = 30522
    hidden: int = 768
    layers: int = 6
    heads: int = 12
    ffn: int = 3072
    type_vocab: int = 1
    head_act: ClassVar[int] = 2

    @staticmethod
    def from_hf(d: dict) -> "DistilBertConfig":
        """config.json of a ``distilbert`` checkpoint -> DistilBertConfig; eps is 1e-12, which DistilBERT hard-codes"""
        if d.get("activation", "gelu") != "gelu":
            raise ValueError(f"distilbert with activation = {d.get('activation')!r} is not supported: only erf-GELU is "
                             f"computed")
        for field in ("vocab_size", "dim", "n_layers", "n_heads", "hidden_dim"):
            if field not in d:
                raise ValueError(f"distilbert config.json without {field!r} is not supported: a DistilBERT checkpoint "
                                 f"states its shape in vocab_size, dim, n_layers, n_heads and hidden_dim")
        return DistilBertConfig(vocab_size=int(d["vocab_size"]), hidden=int(d["dim"]), layers=int(d["n_layers"]),
                                heads=int(d["n_heads"]), ffn=int(d["hidden_dim"]),
                                max_pos=int(d.get("max_position_embeddings", 512)),
                                num_labels=len(d["id2label"]) if "id2label" in d else d.get("num_labels", 1))


# DistilBERT checkpoint names -> the BERT names of ``weight_names`` (the embeddings have BERT's names already)
_DISTILBERT_RENAME = (("transformer.layer.", "encoder.layer."), ("attention.q_lin.", "attention.self.query."),
                      ("attention.k_lin.", "attention.self.key."), ("attention.v_lin.", "attention.self.value."),
                      ("attention.out_lin.", "attention.output.dense."), ("sa_layer_norm.", "attention.output.LayerNorm."),
                      ("ffn.lin1.", "intermediate.dense."), ("ffn.lin2.", "output.dense."),
                      ("output_layer_norm.", "output.LayerNorm."), ("pre_classifier.", "pooler.dense."))


def distilbert_to_canonical(raw: Dict[str, np.ndarray], cfg: DistilBertConfig) -> Dict[str, np.ndarray]:
    """DistilBERT tensors (bare, or under ``distilbert.`` as the sequence-classification model saves them) -> the
    canonical names of ``weight_names``, with a zero [1, H] token-type table.  ``position_embeddings.weight`` is read as
    stored, also for ``sinusoidal_pos_embds`` checkpoints (transformers keeps that table in the state dict).  The
    masked-LM head (``vocab_transform``, ``vocab_layer_norm``, ``vocab_projector``) is dropped."""
    w: Dict[str, np.ndarray] = {}
    for k, v in raw.items():
        k = k[11:] if k.startswith("distilbert.") else k
        if k.startswith(("vocab_transform.", "vocab_layer_norm.", "vocab_projector.")):
            continue
        for a, b in _DISTILBERT_RENAME:
            k = k.replace(a, b)
        w[k] = np.ascontiguousarray(v, dtype=np.float32)
    w["embeddings.token_type_embeddings.weight"] = np.zeros((1, cfg.hidden), np.float32)
    return w


XMOD_LANGUAGE_ENV = "RMU_XMOD_LANGUAGE"
SYNTHETIC_LANGUAGES = ("en_XX", "de_DE", "fr_XX")


def select_language(languages, default: Optional[str], where: str) -> str:
    """The X-MOD language an encoder runs: ``$RMU_XMOD_LANGUAGE`` when set, else ``default`` (config.json's
    ``default_language``).  No language at all, or one that is not in ``languages``, is a ValueError, as transformers'
    ``XmodModel.forward`` raises one without ``lang_ids`` or a default language: such a checkpoint is refused like a
    ``model_type`` the encoder does not run."""
    lang = os.environ.get(XMOD_LANGUAGE_ENV) or default
    if lang is None:
        raise ValueError(f"{where}: model_type 'xmod' is not supported without an input language: config.json sets no "
                         f"default_language; set {XMOD_LANGUAGE_ENV} to one of {list(languages)}")
    if lang not in languages:
        raise ValueError(f"{where}: model_type 'xmod' is not supported in language {lang!r}: it is not one of the "
                         f"checkpoint's languages {list(languages)}")
    return lang


def xmod_languages(d: dict) -> Tuple[str, ...]:
    """config.json's ``languages``, in adapter order (transformers' XmodConfig default: en_XX alone)"""
    return tuple(str(x) for x in d.get("languages", ("en_XX",)))


@dataclass
class XmodConfig(XLMRConfig):
    """X-MOD (transformers ``XmodModel``): XLM-R with a bottleneck adapter per language in every layer, after the
    feed-forward output.  With the flags of ``facebook/xmod-base`` (post-LN, ``adapter_reuse_layer_norm``,
    ``ln_before_adapter``, no adapter LayerNorm) a layer ends ``h = LN(y); out = LN(D2 gelu(D1 h + d1) + d2 + h)`` with
    the layer's own output LayerNorm both times.  One encoder runs one language, ``language``, of ``languages`` (the
    order of ``config.languages``); only that language's adapters are read and uploaded."""
    adapter_dim: int = 384
    languages: Tuple[str, ...] = SYNTHETIC_LANGUAGES
    language: str = SYNTHETIC_LANGUAGES[0]

    @staticmethod
    def from_hf(d: dict, where: str = "xmod") -> "XmodConfig":
        for key, default, want in (("pre_norm", False, False), ("adapter_layer_norm", False, False),
                                   ("adapter_reuse_layer_norm", True, True), ("ln_before_adapter", True, True)):
            if bool(d.get(key, default)) != want:
                raise ValueError(f"xmod with {key} = {d.get(key)} is not supported: the encoder runs X-MOD with "
                                 f"pre_norm false, adapter_layer_norm false, adapter_reuse_layer_norm true and "
                                 f"ln_before_adapter true (facebook/xmod-base's flags)")
        H, r = int(d["hidden_size"]), int(d.get("adapter_reduction_factor", 2))
        if r <= 0 or H % r:
            raise ValueError(f"xmod: hidden_size {H} is not divisible by adapter_reduction_factor {r}")
        base = XLMRConfig.from_hf({**d, "model_type": "xmod"})
        languages = xmod_languages(d)
        lang = select_language(languages, d.get("default_language"), where)
        return XmodConfig(**asdict(base), adapter_dim=H // r, languages=languages, language=lang)


@dataclass
class DebertaConfig(BertConfig):
    """DeBERTa-v2 / v3 (transformers ``DebertaV2Model``; mxbai-rerank-*-v1, cross-encoder/nli-deberta-v3-*): BERT's
    post-LN encoder with disentangled attention and no absolute positions or token types.  Every score adds
    ``Q_i . PK[c] + K_j . PQ[c]``, with ``PQ`` / ``PK`` the layer's own query / key projections (biases included) of
    ``R = LN_rel(rel_embeddings[0:2s])`` and ``c = clamp(s + bucket(i - j), 0, 2s - 1)``, and the three terms share the
    scale ``1 / sqrt(3 d_h)``.  The encoder gets zero position [max_pos, H] and token-type [1, H] tables:
    ``(w + 0) + 0 == w`` exactly.  The head is ContextPooler (erf-GELU) + classifier."""
    vocab_size: int = 128100
    max_pos: int = 512
    type_vocab: int = 1
    ln_eps: float = 1e-7
    position_buckets: int = 256
    max_relative_positions: int = 512
    head_act: int = 1

    @staticmethod
    def from_hf(d: dict) -> "DebertaConfig":
        """config.json of a ``deberta-v2`` checkpoint -> DebertaConfig; refuses, naming the field, what the encoder does
        not compute"""
        def refuse(field, why):
            raise ValueError(f"deberta-v2 with {field} = {d.get(field)!r} is not supported: {why}")
        if not d.get("relative_attention", False):
            refuse("relative_attention", "the encoder runs DeBERTa with relative (disentangled) attention only")
        if int(d.get("position_buckets", -1)) <= 0:
            refuse("position_buckets", "the encoder runs log-bucketed relative positions (position_buckets > 0) only")
        if not d.get("share_att_key", False):
            refuse("share_att_key", "the position projections are the layer's own query / key projections")
        pat = d.get("pos_att_type") or []
        pat = pat.split("|") if isinstance(pat, str) else list(pat)
        if sorted(x.strip().lower() for x in pat) != ["c2p", "p2c"]:
            refuse("pos_att_type", "the encoder computes exactly the c2p and p2c terms")
        if "layer_norm" not in [x.strip() for x in str(d.get("norm_rel_ebd", "none")).lower().split("|")]:
            refuse("norm_rel_ebd", "the relative embeddings must pass the encoder's LayerNorm (layer_norm)")
        if d.get("position_biased_input", True):
            refuse("position_biased_input", "DeBERTa-v3 adds no absolute positions")
        if int(d.get("type_vocab_size", 0)) > 0:
            refuse("type_vocab_size", "DeBERTa-v3 has no token types")
        if int(d.get("conv_kernel_size", 0)) > 0:
            refuse("conv_kernel_size", "the ConvLayer of deberta-v2-xlarge is not computed")
        H = int(d["hidden_size"])
        if int(d.get("embedding_size", H)) != H:
            refuse("embedding_size", f"it must equal hidden_size {H} (no embed_proj)")
        for key in ("hidden_act", "pooler_hidden_act"):
            if d.get(key, "gelu") != "gelu":
                refuse(key, "only erf-GELU is computed")
        max_pos = int(d.get("max_position_embeddings", 512))
        mrp = int(d.get("max_relative_positions", -1))
        return DebertaConfig(vocab_size=d["vocab_size"], hidden=H, layers=d["num_hidden_layers"],
                             heads=d["num_attention_heads"], ffn=d["intermediate_size"], max_pos=max_pos,
                             ln_eps=d.get("layer_norm_eps", 1e-7),
                             num_labels=len(d["id2label"]) if "id2label" in d else d.get("num_labels", 1),
                             position_buckets=int(d["position_buckets"]),
                             max_relative_positions=mrp if mrp >= 1 else max_pos)


def modernbert_windows(layers: int, global_every: int = 3, local_attention: int = 128) -> Tuple[int, ...]:
    """per-layer half-windows of ModernBERT's release config form: layer l is global (0) when l % global_every == 0,
    else local with half-window local_attention // 2"""
    return tuple(0 if l % global_every == 0 else local_attention // 2 for l in range(layers))


@dataclass
class ModernBertConfig(BertConfig):
    """ModernBERT (transformers ``ModernBertModel`` / ``ModernBertForSequenceClassification``; gte-reranker-modernbert,
    modernbert-embed, gte-modernbert): a pre-LN encoder, ``x += Wo attn(LN_a(x))``, ``x += Wo mlp(LN_m(x))``, then
    ``final_norm``, with ``LN_a`` the identity in layer 0.  Rotary positions on q and k (``global_theta`` on global
    layers, ``local_theta`` on local ones, no position table), a GeGLU feed-forward (``Wi`` [2F, H]: ``gelu(input) *
    gate``), sliding-window attention ``|i - j| <= layer_windows[l]`` on the local layers (0 = global), and the head
    ``classifier(LN(gelu(dense(p))))`` on the CLS row or the mean of the final hidden state (``classifier_pooling``).
    Absent biases and LayerNorm shifts are zero tensors in the weight dict."""
    vocab_size: int = 50368
    hidden: int = 768
    layers: int = 22
    heads: int = 12
    ffn: int = 1152
    max_pos: int = 8192
    type_vocab: int = 1
    ln_eps: float = 1e-5
    layer_windows: Tuple[int, ...] = ()
    global_theta: float = 160000.0
    local_theta: float = 10000.0
    classifier_pooling: str = "cls"

    def __post_init__(self):
        if not self.layer_windows:
            self.layer_windows = modernbert_windows(self.layers)
        self.layer_windows = tuple(int(x) for x in self.layer_windows)
        if len(self.layer_windows) != self.layers:
            raise ValueError(f"modernbert: {len(self.layer_windows)} layer windows for {self.layers} layers")

    @staticmethod
    def from_hf(d: dict) -> "ModernBertConfig":
        """config.json of a ``modernbert`` checkpoint, in the release form (``global_attn_every_n_layers``,
        ``global_rope_theta``, ``local_rope_theta``, ``local_attention``) or transformers 5's (``layer_types``,
        ``rope_parameters``) -> ModernBertConfig; refuses, naming the field, what the encoder does not compute"""
        def refuse(field, value, why):
            raise ValueError(f"modernbert with {field} = {value!r} is not supported: {why}")
        for key in ("hidden_activation", "classifier_activation"):
            if d.get(key, "gelu") != "gelu":
                refuse(key, d.get(key), "only erf-GELU is computed")
        pooling = d.get("classifier_pooling", "cls")
        if pooling not in ("cls", "mean"):
            refuse("classifier_pooling", pooling, "the head pools by cls or mean")
        H, nh, L = int(d["hidden_size"]), int(d["num_attention_heads"]), int(d["num_hidden_layers"])
        if d.get("head_dim") is not None and int(d["head_dim"]) != H // nh:
            refuse("head_dim", d["head_dim"], f"it must be hidden_size / num_attention_heads = {H // nh}")
        half = int(d.get("local_attention", 128)) // 2
        types = d.get("layer_types")
        if types:
            if len(types) != L:
                refuse("layer_types", types, f"it must name {L} layers")
            for t in types:
                if t not in ("full_attention", "sliding_attention"):
                    refuse("layer_types", t, "layers are full_attention or sliding_attention")
            windows = tuple(0 if t == "full_attention" else half for t in types)
        else:
            windows = modernbert_windows(L, int(d.get("global_attn_every_n_layers", 3)), 2 * half)
        theta = {"full_attention": float(d.get("global_rope_theta", 160000.0)),
                 "sliding_attention": float(d.get("local_rope_theta", 10000.0))}
        if d.get("rope_scaling"):
            refuse("rope_scaling", d["rope_scaling"], "RoPE scaling is not computed")
        rp = d.get("rope_parameters")
        if rp:
            for t in theta:
                p = rp.get(t, rp) or {}
                if p.get("rope_type", "default") != "default":
                    refuse("rope_type", p.get("rope_type"), "only the default rotary embedding is computed")
                if p.get("rope_theta") is not None:
                    theta[t] = float(p["rope_theta"])
        return ModernBertConfig(vocab_size=int(d["vocab_size"]), hidden=H, layers=L, heads=nh,
                                ffn=int(d["intermediate_size"]), max_pos=int(d.get("max_position_embeddings", 8192)),
                                ln_eps=float(d.get("norm_eps", 1e-5)),
                                num_labels=len(d["id2label"]) if "id2label" in d else d.get("num_labels", 1),
                                layer_windows=windows, global_theta=theta["full_attention"],
                                local_theta=theta["sliding_attention"], classifier_pooling=pooling)


def rope_tables(cfg: ModernBertConfig):
    """(cos_global, sin_global, cos_local, sin_local), each [max_pos, d_h / 2] float32, as transformers'
    ``ModernBertRotaryEmbedding`` computes them: ``inv_freq = 1 / (theta ** (arange(0, d, 2).float() / d))``, the angle
    ``pos * inv_freq`` in float32, then ``.cos()`` / ``.sin()``.  At pos ~ 8000 one float32 ulp of the angle is ~5e-4 rad,
    so these float32 tables define the model: the float64 oracle looks its cos / sin up in them too."""
    return (*rope_table(cfg.global_theta, cfg.head_dim, cfg.max_pos), *rope_table(cfg.local_theta, cfg.head_dim, cfg.max_pos))


def rope_table(theta: float, head_dim: int, rows: int, llama3: Optional[Tuple[float, float, float, int]] = None):
    """(cos, sin), each [rows, head_dim / 2] float32, of the default rotary embedding as transformers computes it
    (``ModernBertRotaryEmbedding``, ``Qwen3RotaryEmbedding``): ``inv_freq = 1 / (theta ** (arange(0, d, 2).float() /
    d))``, the angle ``pos * inv_freq`` in float32, then ``.cos()`` / ``.sin()``.  ``llama3`` = (factor, low_freq_factor,
    high_freq_factor, original_max_position_embeddings) applies Llama-3.1's frequency scaling to inv_freq first, in
    float32 as transformers' ``llama3`` rope init does: wavelengths 2 pi / inv_freq above old / low_freq_factor are
    divided by factor, those below old / high_freq_factor kept, and those between interpolated."""
    import math
    import torch
    d = head_dim
    pos = torch.arange(rows, dtype=torch.int64).float()
    inv_freq = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.int64).float() / d))
    if llama3 is not None:
        factor, low, high, old = llama3
        wavelen = 2 * math.pi / inv_freq
        scaled = torch.where(wavelen > old / low, inv_freq / factor, inv_freq)
        smooth = (old / wavelen - low) / (high - low)
        smoothed = (1 - smooth) * scaled / factor + smooth * scaled
        medium = ~(wavelen < old / high) * ~(wavelen > old / low)
        inv_freq = torch.where(medium, smoothed, scaled)
    ang = pos[:, None] * inv_freq[None, :]
    return (np.ascontiguousarray(ang.cos().numpy(), dtype=np.float32),
            np.ascontiguousarray(ang.sin().numpy(), dtype=np.float32))


def modernbert_weight_names(cfg: ModernBertConfig, with_head: bool):
    """canonical ModernBERT tensors (transformers' names without ``model.``) in rmu_encoder_create_modernbert's order;
    ``layers.0.attn_norm.*`` are placeholders (ones, zeros) that the encoder does not read"""
    H, F = cfg.hidden, cfg.ffn
    names = [("embeddings.tok_embeddings.weight", (cfg.vocab_size, H)), ("embeddings.norm.weight", (H,)),
             ("embeddings.norm.bias", (H,))]
    for l in range(cfg.layers):
        p = f"layers.{l}."
        names += [(p + "attn_norm.weight", (H,)), (p + "attn_norm.bias", (H,)),
                  (p + "attn.Wqkv.weight", (3 * H, H)), (p + "attn.Wqkv.bias", (3 * H,)),
                  (p + "attn.Wo.weight", (H, H)), (p + "attn.Wo.bias", (H,)),
                  (p + "mlp_norm.weight", (H,)), (p + "mlp_norm.bias", (H,)),
                  (p + "mlp.Wi.weight", (2 * F, H)), (p + "mlp.Wi.bias", (2 * F,)),
                  (p + "mlp.Wo.weight", (H, F)), (p + "mlp.Wo.bias", (H,))]
    names += [("final_norm.weight", (H,)), ("final_norm.bias", (H,))]
    if with_head:
        names += [("head.dense.weight", (H, H)), ("head.dense.bias", (H,)), ("head.norm.weight", (H,)),
                  ("head.norm.bias", (H,)), ("classifier.weight", (cfg.num_labels, H)),
                  ("classifier.bias", (cfg.num_labels,))]
    return names


def modernbert_to_canonical(raw: Dict[str, np.ndarray], cfg: ModernBertConfig, with_head: bool) -> Dict[str, np.ndarray]:
    """ModernBERT tensors (under ``model.``, as both transformers classes save them, or bare) plus ``head.*`` /
    ``classifier.*`` -> the names of ``modernbert_weight_names``.  Zero vectors stand in for the biases and LayerNorm
    shifts a checkpoint does not have (``attention_bias``, ``mlp_bias``, ``norm_bias`` and ``classifier_bias`` false),
    and ones / zeros for layer 0's absent ``attn_norm``.  The masked-LM head (``head.*`` without a classifier, and
    ``decoder.*``) is dropped."""
    w: Dict[str, np.ndarray] = {}
    for k, v in raw.items():
        if k.startswith("decoder.") or (not with_head and k.startswith("head.")):
            continue
        k = k[6:] if k.startswith("model.") else k
        w[k] = np.ascontiguousarray(v, dtype=np.float32)
    for name, shape in modernbert_weight_names(cfg, with_head):
        if name not in w and (name.endswith(".bias") or name == "layers.0.attn_norm.weight"):
            w[name] = (np.ones if name.endswith("attn_norm.weight") else np.zeros)(shape, np.float32)
    return w


@dataclass
class Qwen3Config(BertConfig):
    """Qwen3 (transformers ``Qwen3Model`` / ``Qwen3ForSequenceClassification`` / ``Qwen3ForCausalLM``; Qwen3-Embedding,
    Qwen3-Reranker): a decoder run as an encoder.  RMSNorm (``w * (x * rsqrt(mean(x^2) + eps))``), grouped-query causal
    attention with ``kv_heads`` key / value heads of ``head_dim`` (128), per-head RMSNorm of q and k, rotary positions
    (``rope_theta``), a SwiGLU feed-forward and no biases.  Its outputs take one row per sequence: the last token
    (embedders), or with a head the rightmost token whose id != ``pad_token_id`` (``Qwen3ForSequenceClassification``)
    or the last token (the causal-LM reranker, ``head_pad_id`` -1).  ``head`` in the weight dict is the [num_labels, H]
    last-token head; ``name`` names the model in errors."""
    vocab_size: int = 151669
    hidden: int = 1024
    layers: int = 28
    heads: int = 16
    ffn: int = 3072
    max_pos: int = 40960
    type_vocab: int = 1
    ln_eps: float = 1e-6
    kv_heads: int = 8
    head_dim: int = 128
    rope_theta: float = 1000000.0
    tie_word_embeddings: bool = True
    pad_token_id: Optional[int] = None
    name: str = "qwen3"
    reranker: bool = False      # a Qwen3ForCausalLM reranker: head = the [no, yes] rows of lm_head, read at the last token
    prompt: str = ""            # the embedder's default prompt (config_sentence_transformers.json), prepended to texts

    @property
    def head_pad_id(self) -> int:
        """the id the last-token head skips from the right: ``pad_token_id`` (sequence classification); -1 (the last
        token) for the causal-LM reranker or without a pad id"""
        return -1 if self.reranker or self.pad_token_id is None else int(self.pad_token_id)

    @staticmethod
    def from_hf(d: dict, name: str = "qwen3") -> "Qwen3Config":
        """config.json of a ``qwen3`` checkpoint -> Qwen3Config; refuses, naming the field, what the encoder does not
        compute"""
        def refuse(field, value, why):
            raise ValueError(f"{name}: qwen3 with {field} = {value!r} is not supported: {why}")
        if d.get("model_type", "qwen3") != "qwen3":
            refuse("model_type", d.get("model_type"), "only model_type 'qwen3' runs as Qwen3 (not MoE or Qwen2)")
        if d.get("hidden_act", "silu") != "silu":
            refuse("hidden_act", d.get("hidden_act"), "only SwiGLU (silu) is computed")
        if d.get("attention_bias", False):
            refuse("attention_bias", d["attention_bias"], "q / k / v / o have no biases in the encoder")
        if d.get("use_sliding_window", False):
            refuse("use_sliding_window", d["use_sliding_window"], "only full causal attention is computed")
        for t in d.get("layer_types") or ():
            if t != "full_attention":
                refuse("layer_types", t, "only full_attention layers are computed")
        if d.get("rope_scaling"):
            refuse("rope_scaling", d["rope_scaling"], "RoPE scaling is not computed")
        rp = d.get("rope_parameters") or {}
        if rp.get("rope_type", "default") != "default":
            refuse("rope_type", rp.get("rope_type"), "only the default rotary embedding is computed")
        theta = rp.get("rope_theta", d.get("rope_theta", 10000.0))
        H, nh = int(d["hidden_size"]), int(d["num_attention_heads"])
        pad = d.get("pad_token_id")
        return Qwen3Config(vocab_size=int(d["vocab_size"]), hidden=H, layers=int(d["num_hidden_layers"]), heads=nh,
                           ffn=int(d["intermediate_size"]), max_pos=int(d.get("max_position_embeddings", 40960)),
                           ln_eps=float(d.get("rms_norm_eps", 1e-6)),
                           num_labels=len(d["id2label"]) if "id2label" in d else d.get("num_labels", 1),
                           kv_heads=int(d.get("num_key_value_heads") or nh), head_dim=int(d.get("head_dim") or H // nh),
                           rope_theta=float(theta), tie_word_embeddings=bool(d.get("tie_word_embeddings", False)),
                           pad_token_id=None if pad is None else int(pad), name=name)


def qwen3_weight_names(cfg: Qwen3Config, with_head: bool):
    """canonical Qwen3 tensors (transformers' names without ``model.``) in rmu_encoder_create_qwen3's order; ``head``
    [num_labels, H] is the last-token head (``score.weight``, or the yes / no rows of ``lm_head``)"""
    H, F, d = cfg.hidden, cfg.ffn, cfg.head_dim
    names = [("embed_tokens.weight", (cfg.vocab_size, H))]
    for l in range(cfg.layers):
        p = f"layers.{l}."
        names += [(p + "input_layernorm.weight", (H,)), (p + "self_attn.q_proj.weight", (cfg.heads * d, H)),
                  (p + "self_attn.k_proj.weight", (cfg.kv_heads * d, H)),
                  (p + "self_attn.v_proj.weight", (cfg.kv_heads * d, H)), (p + "self_attn.q_norm.weight", (d,)),
                  (p + "self_attn.k_norm.weight", (d,)), (p + "self_attn.o_proj.weight", (H, cfg.heads * d)),
                  (p + "post_attention_layernorm.weight", (H,)), (p + "mlp.gate_proj.weight", (F, H)),
                  (p + "mlp.up_proj.weight", (F, H)), (p + "mlp.down_proj.weight", (H, F))]
    names.append(("norm.weight", (H,)))
    if with_head:
        names.append(("head", (cfg.num_labels, H)))
    return names


def qwen3_to_canonical(raw: Dict[str, np.ndarray], cfg: Qwen3Config) -> Dict[str, np.ndarray]:
    """Qwen3 tensors under ``model.`` (as every transformers class saves them) or bare -> the names of
    ``qwen3_weight_names``; ``score.weight`` (sequence classification) becomes ``head``, ``lm_head.weight`` is dropped
    (the reranker reads its two rows itself)."""
    w: Dict[str, np.ndarray] = {}
    for k, v in raw.items():
        if k == "lm_head.weight":
            continue
        k = "head" if k == "score.weight" else (k[6:] if k.startswith("model.") else k)
        w[k] = np.ascontiguousarray(v, dtype=np.float32)
    return w


def _synthetic_draw(rng: np.random.Generator, name: str, shape, scale: float) -> np.ndarray:
    """one seeded decoder tensor from ``rng``'s stream: norm weights 1 + N(0, 0.1), embeddings N(0, 0.02) (three times
    that when scale > 1), everything else N(0, 0.02 scale)"""
    if name.endswith("norm.weight") or name.endswith("layernorm.weight"):
        a = 1.0 + 0.1 * rng.standard_normal(shape)
    elif name == "embed_tokens.weight":
        a = 0.02 * rng.standard_normal(shape) * (3.0 if scale > 1 else 1.0)
    else:
        a = 0.02 * scale * rng.standard_normal(shape)
    return np.ascontiguousarray(a, dtype=np.float32)


def synthetic_qwen3_weights(cfg: Qwen3Config, seed: int = 0, with_head: bool = False,
                            scale: float = 1.0) -> Dict[str, np.ndarray]:
    """seeded Qwen3 weights: projections N(0, 0.02 scale), norm weights near 1, embeddings N(0, 0.02) (transformers'
    init, with norm gains spread so a wrong weight layout shows in the numbers)"""
    rng = np.random.default_rng(seed)
    return {name: _synthetic_draw(rng, name, shape, scale) for name, shape in qwen3_weight_names(cfg, with_head)}


def qwen3_lm_rows(path: str, cfg: Qwen3Config, ids) -> np.ndarray:
    """rows ``ids`` of ``lm_head.weight`` (``embed_tokens`` when the embeddings are tied or the head is absent), read
    one row at a time from the snapshot's safetensors -> float32 [len(ids), H]"""
    import torch
    from safetensors import safe_open
    names = ["lm_head.weight"] if not cfg.tie_word_embeddings else []
    names += ["model.embed_tokens.weight", "embed_tokens.weight"]
    files = _safetensors_files(path)
    for name in names:
        for f in files:
            with safe_open(f, framework="pt") as fh:
                if name in fh.keys():
                    sl = fh.get_slice(name)
                    return np.stack([sl[int(i):int(i) + 1].to(torch.float32).numpy()[0] for i in ids]).astype(np.float32)
    raise KeyError(f"{path}: no lm_head.weight or embed_tokens.weight to read the reranker's yes / no rows from")


@dataclass
class LlamaConfig(BertConfig):
    """Llama-3 (transformers ``LlamaModel``, model_type ``llama``): Qwen3's decoder without the per-head q / k RMSNorm,
    with ``llama3`` rope scaling (``rope_scaling`` = (factor, low_freq_factor, high_freq_factor,
    original_max_position_embeddings)) or the default rotary embedding (``rope_scaling`` None).  It runs for attention
    provenance and generation only (``provenance.DecoderAttention``), never as an embedder or reranker; ``lm_head`` is
    read by ``decoder_lm_head`` when generation first runs.
    Defaults: the Llama-3.1-8B shape."""
    vocab_size: int = 128256
    hidden: int = 4096
    layers: int = 32
    heads: int = 32
    ffn: int = 14336
    max_pos: int = 131072
    type_vocab: int = 1
    ln_eps: float = 1e-5
    kv_heads: int = 8
    head_dim: int = 128
    rope_theta: float = 500000.0
    rope_scaling: Optional[Tuple[float, float, float, int]] = (8.0, 1.0, 4.0, 8192)
    name: str = "llama"

    def rope_tables(self):
        return rope_table(self.rope_theta, self.head_dim, self.max_pos, self.rope_scaling)

    @staticmethod
    def from_hf(d: dict, name: str = "llama") -> "LlamaConfig":
        """config.json of a ``llama`` checkpoint, with ``rope_scaling`` (the release form) or ``rope_parameters``
        (transformers 5) -> LlamaConfig; refuses, naming the field, what the decoder does not compute"""
        def refuse(field, value, why):
            raise ValueError(f"{name}: llama with {field} = {value!r} is not supported: {why}")
        if d.get("model_type", "llama") != "llama":
            refuse("model_type", d.get("model_type"), "only model_type 'llama' runs as Llama")
        if d.get("hidden_act", "silu") != "silu":
            refuse("hidden_act", d.get("hidden_act"), "only SwiGLU (silu) is computed")
        for field in ("attention_bias", "mlp_bias"):
            if d.get(field, False):
                refuse(field, d[field], "the projections have no biases in the decoder")
        rp = d.get("rope_parameters") or d.get("rope_scaling") or {}
        kind = rp.get("rope_type", rp.get("type", "default"))
        if kind not in ("default", "llama3"):
            refuse("rope_type", kind, "only the default and llama3 rotary embeddings are computed")
        theta = float(rp.get("rope_theta", d.get("rope_theta", 10000.0)))
        H, nh = int(d["hidden_size"]), int(d["num_attention_heads"])
        hd = int(d.get("head_dim") or H // nh)
        if hd != 128:
            refuse("head_dim", hd, "the decoder's attention kernels take head_dim 128 only")
        max_pos = int(d.get("max_position_embeddings", 2048))
        scaling = None
        if kind == "llama3":
            scaling = (float(rp["factor"]), float(rp["low_freq_factor"]), float(rp["high_freq_factor"]),
                       int(rp.get("original_max_position_embeddings") or max_pos))
        return LlamaConfig(vocab_size=int(d["vocab_size"]), hidden=H, layers=int(d["num_hidden_layers"]), heads=nh,
                           ffn=int(d["intermediate_size"]), max_pos=max_pos, ln_eps=float(d.get("rms_norm_eps", 1e-6)),
                           kv_heads=int(d.get("num_key_value_heads") or nh), head_dim=hd, rope_theta=theta,
                           rope_scaling=scaling, name=name)


def llama_weight_names(cfg: LlamaConfig):
    """canonical Llama tensors (transformers' names without ``model.``) in rmu_encoder_create_llama's order"""
    drop = (".self_attn.q_norm.weight", ".self_attn.k_norm.weight")
    return [(n, shape) for n, shape in qwen3_weight_names(cfg, False) if not n.endswith(drop)]


def synthetic_llama_weights(cfg: LlamaConfig, seed: int = 0, scale: float = 1.0) -> Dict[str, np.ndarray]:
    """seeded Llama weights, drawn as ``synthetic_qwen3_weights`` draws them"""
    rng = np.random.default_rng(seed)
    return {name: _synthetic_draw(rng, name, shape, scale) for name, shape in llama_weight_names(cfg)}


# decoders for attention provenance (provenance.DecoderAttention), apart from PRESETS: the embedders, rerankers and
# ColBERT never take them.  tiny-llama: head_dim 128, two query heads per kv head, three layers, and llama3 scaling
# with original_max_position_embeddings 64, so that several of its frequencies are divided or interpolated.
# llama-3.1-8b: Meta-Llama-3.1-8B-Instruct's shape [3P-recall: its config.json is not read here].
# llama-3.1-70b: Llama-3.1-70B-Instruct's (and Llama-3.3-70B-Instruct's) shape, and qwen3-32b: Qwen3-32B's
# [3P-recall: their config.json files are not read here]; both run in NF4 only (hidden above 4096).
# Draft models for speculative decoding (DecoderAttention.generate's assistant), sharing their targets' vocabularies:
# llama-3.2-3b: Llama-3.2-3B-Instruct's shape, tied embeddings and llama3 rope scaling factor 32, the draft of
# Llama-3.1-8B / 70B and Llama-3.3-70B; qwen3-0.6b: Qwen3-0.6B's shape as a chat decoder (vocabulary 151936, tied
# embeddings), the draft of Qwen3-8B / 14B / 32B [3P-recall: their config.json files are not read here].  A synthetic
# preset's LM head is drawn on its own, so the tie only matters for snapshots (decoder_lm_head reads it there).
# tiny-llama-draft: one layer, two query heads over one kv head, with tiny-llama's vocabulary and rope.
DECODER_PRESETS: Dict[str, BertConfig] = {
    "tiny-llama": LlamaConfig(vocab_size=1000, hidden=256, layers=3, heads=4, ffn=384, max_pos=8192, kv_heads=2,
                              rope_theta=10000.0, rope_scaling=(8.0, 1.0, 4.0, 64)),
    "tiny-llama-draft": LlamaConfig(vocab_size=1000, hidden=256, layers=1, heads=2, ffn=384, max_pos=8192, kv_heads=1,
                                    rope_theta=10000.0, rope_scaling=(8.0, 1.0, 4.0, 64)),
    "llama-3.2-3b": LlamaConfig(hidden=3072, layers=28, heads=24, ffn=8192, kv_heads=8,
                                rope_scaling=(32.0, 1.0, 4.0, 8192)),
    "qwen3-0.6b": Qwen3Config(vocab_size=151936, hidden=1024, layers=28, heads=16, ffn=3072, kv_heads=8,
                              tie_word_embeddings=True, num_labels=1),
    "llama-3.1-8b": LlamaConfig(),
    "llama-3.1-70b": LlamaConfig(hidden=8192, layers=80, heads=64, ffn=28672),
    "qwen3-32b": Qwen3Config(vocab_size=151936, hidden=5120, layers=64, heads=64, ffn=25600, kv_heads=8,
                             tie_word_embeddings=False, num_labels=1),
}


def _decoder_config_of_snapshot(path: str) -> BertConfig:
    cfgd = _read_json(os.path.join(path, "config.json"))
    if cfgd is None:
        raise FileNotFoundError(f"{path}: no config.json")
    kind = cfgd.get("model_type")
    if kind == "llama":
        return LlamaConfig.from_hf(cfgd, name=path)
    if kind == "qwen3":
        return Qwen3Config.from_hf(cfgd, name=path)
    raise ValueError(f"{path}: model_type {kind!r} is not supported for attention provenance (llama, qwen3)")


def decoder_weight_names(cfg: BertConfig):
    """``llama_weight_names`` or, for a Qwen3 config, ``qwen3_weight_names`` without a head"""
    return llama_weight_names(cfg) if isinstance(cfg, LlamaConfig) else qwen3_weight_names(cfg, False)


def _load_decoder_snapshot(path: str):
    """a ``llama`` or ``qwen3`` snapshot -> (config, weights) of the decoder without any head; ``lm_head`` (and a
    sequence-classification ``score``) is never read"""
    cfg = _decoder_config_of_snapshot(path)
    names = decoder_weight_names(cfg)
    w = qwen3_to_canonical(_load_tensors(path, lambda n: n not in ("lm_head.weight", "score.weight")), cfg)
    missing = [n for n, _ in names if n not in w]
    if missing:
        raise KeyError(f"{path}: missing tensors {missing[:4]}...")
    return cfg, {n: w[n] for n, _ in names}


def resolve_decoder(model_name: str, cache_folder: Optional[str] = None):
    """decoder name -> (config, weights): ``synthetic:<preset>[:seed[:scale]]`` (DECODER_PRESETS, or a Qwen3 preset of
    PRESETS), else a local snapshot directory found as ``resolve_model`` finds one"""
    if model_name.startswith("synthetic:"):
        parts = model_name.split(":")
        preset = parts[1]
        seed = int(parts[2]) if len(parts) > 2 else 0
        scale = float(parts[3]) if len(parts) > 3 else 1.0
        cfg = decoder_config(model_name)
        if isinstance(cfg, LlamaConfig):
            return cfg, synthetic_llama_weights(cfg, seed=seed, scale=scale)
        return cfg, synthetic_qwen3_weights(cfg, seed=seed, with_head=False, scale=scale)
    return _load_decoder_snapshot(find_snapshot(model_name, cache_folder))


def decoder_config(model_name: str, cache_folder: Optional[str] = None) -> BertConfig:
    """the config of ``resolve_decoder``'s decoder, read without any tensor: a synthetic preset's, or the snapshot's
    config.json"""
    if model_name.startswith("synthetic:"):
        preset = model_name.split(":")[1]
        if preset in DECODER_PRESETS:
            base = DECODER_PRESETS[preset]
        elif preset in PRESETS and isinstance(PRESETS[preset][0], Qwen3Config):
            base = PRESETS[preset][0]
        else:
            raise ValueError(f"unknown synthetic decoder preset {preset!r}; have {sorted(DECODER_PRESETS)} and the "
                             f"qwen3 presets")
        cfg = type(base)(**asdict(base))
        cfg.name = model_name
        if isinstance(cfg, Qwen3Config):
            cfg.reranker, cfg.num_labels = False, 1
        return cfg
    return _decoder_config_of_snapshot(find_snapshot(model_name, cache_folder))


class DecoderLayers:
    """A decoder's weights read one layer at a time (``rmu_decoder_create_nf4`` / ``rmu_decoder_load_layer_nf4``):
    ``cfg``; ``globals()`` -> embed_tokens and the final norm; ``layer(l)`` -> layer l's tensors in
    ``decoder_weight_names`` order (canonical names, float32).  Host memory holds the embeddings and one layer."""

    def __init__(self, cfg: BertConfig):
        self.cfg = cfg

    def globals(self) -> Dict[str, np.ndarray]:
        raise NotImplementedError

    def layer(self, l: int) -> Dict[str, np.ndarray]:
        raise NotImplementedError

    def layer_names(self, l: int):
        p = f"layers.{l}."
        return [(n, shape) for n, shape in decoder_weight_names(self.cfg) if n.startswith(p)]


class DictDecoderLayers(DecoderLayers):
    """the layered view of a whole weight dict (``resolve_decoder``'s)"""

    def __init__(self, cfg: BertConfig, w: Dict[str, np.ndarray]):
        super().__init__(cfg)
        self.w = w

    def globals(self):
        return {n: self.w[n] for n in ("embed_tokens.weight", "norm.weight")}

    def layer(self, l):
        return {n: self.w[n] for n, _ in self.layer_names(l)}


class SyntheticDecoderLayers(DecoderLayers):
    """``synthetic:<preset>[:seed[:scale]]`` drawn one layer at a time: the same tensors, bit for bit, as
    ``synthetic_llama_weights`` / ``synthetic_qwen3_weights``, whose one seeded stream runs embeddings, layers 0 ..
    L - 1, final norm.  The final norm is needed first, so ``globals`` walks the whole stream once, drawing each layer
    and dropping it, and keeps only the generator's state at every layer's start; ``layer(l)`` then draws layer l again
    from its state.  Every layer is therefore drawn twice, on the host in float64 (for a synthetic 70B about 68 G
    normals each time: minutes, not seconds); ``tools/bench_generate.py`` draws its 70B weights on the device instead.
    Nothing but those states is kept between calls."""

    def __init__(self, cfg: BertConfig, seed: int = 0, scale: float = 1.0):
        super().__init__(cfg)
        self.seed, self.scale = seed, scale
        self._states: list = []

    def globals(self):
        rng = np.random.default_rng(self.seed)
        names = decoder_weight_names(self.cfg)
        out = {names[0][0]: _synthetic_draw(rng, *names[0], self.scale)}
        states = []
        for l in range(self.cfg.layers):
            states.append(rng.bit_generator.state)
            for n, shape in self.layer_names(l):
                _synthetic_draw(rng, n, shape, self.scale)
        out[names[-1][0]] = _synthetic_draw(rng, *names[-1], self.scale)
        self._states = states
        return out

    def layer(self, l):
        if not self._states:
            self.globals()
        rng = np.random.default_rng()
        rng.bit_generator.state = self._states[l]
        return {n: _synthetic_draw(rng, n, shape, self.scale) for n, shape in self.layer_names(l)}


class SnapshotDecoderLayers(DecoderLayers):
    """a ``llama`` or ``qwen3`` snapshot read with safetensors' ``safe_open``, tensor by tensor, from
    ``model.safetensors`` or the shards ``model.safetensors.index.json`` lists; bfloat16 is widened to float32 (exact)"""

    def __init__(self, path: str):
        super().__init__(_decoder_config_of_snapshot(path))
        self.path = path
        idx = _read_json(os.path.join(path, SHARD_INDEX))
        single = os.path.join(path, "model.safetensors")
        if os.path.exists(single) or idx is None:
            from safetensors import safe_open
            with safe_open(single, framework="pt") as f:
                self.where = {k: single for k in f.keys()}
        else:
            self.where = {k: os.path.join(path, f) for k, f in idx["weight_map"].items()}

    def _read(self, names) -> Dict[str, np.ndarray]:
        import torch
        from safetensors import safe_open
        stored = {}
        for n in names:
            for k in ("model." + n, n):
                if k in self.where:
                    stored[n] = k
                    break
            else:
                raise KeyError(f"{self.path}: missing tensor {n}")
        out: Dict[str, np.ndarray] = {}
        for f in dict.fromkeys(self.where[k] for k in stored.values()):
            with safe_open(f, framework="pt") as fh:
                for n, k in stored.items():
                    if self.where[k] == f:
                        out[n] = np.ascontiguousarray(fh.get_tensor(k).to(torch.float32).numpy())
        return {n: out[n] for n in names}

    def globals(self):
        return self._read(["embed_tokens.weight", "norm.weight"])

    def layer(self, l):
        return self._read([n for n, _ in self.layer_names(l)])


def decoder_layers(model_name: str, cache_folder: Optional[str] = None) -> DecoderLayers:
    """``resolve_decoder``'s decoder as a ``DecoderLayers``: the same tensors, read or drawn one layer at a time"""
    if model_name.startswith("synthetic:"):
        parts = model_name.split(":")
        return SyntheticDecoderLayers(decoder_config(model_name), seed=int(parts[2]) if len(parts) > 2 else 0,
                                      scale=float(parts[3]) if len(parts) > 3 else 1.0)
    path = find_snapshot(model_name, cache_folder)
    if not _safetensors_snapshot(path):
        # a snapshot that ships only pytorch_model.bin: a pickle cannot be read tensor by tensor, so it is read whole
        # (with weights_only, as _load_tensors reads it) and handed over layer by layer
        return DictDecoderLayers(*_load_decoder_snapshot(path))
    return SnapshotDecoderLayers(path)


def _safetensors_snapshot(path: str) -> bool:
    """``model.safetensors`` or a sharded safetensors index is present"""
    return os.path.exists(os.path.join(path, "model.safetensors")) or os.path.exists(os.path.join(path, SHARD_INDEX))


GB = 1e9
SPLIT_MAX_HIDDEN = 4096           # rmu_encoder_create_llama / _qwen3: split planes stop here; NF4 goes to 8192
NF4_LOAD_STAGING = (1 << 24) * 6  # rmu_decoder_load_layer_nf4's staging chunk: 16 Mi fp32 values and their lo plane


def decoder_memory_plan(cfg: BertConfig, weights: str) -> Dict[str, int]:
    """the device bytes a decoder handle holds once built, computed from the config alone: ``layers`` (the projections:
    NF4 codes + absmax, or split planes), ``embeddings`` (fp32), ``lm_head`` (split planes, attached at the first
    generation), ``scratch`` (NF4's prefill plane pair, the size of the largest projection), ``other`` (norms, rope
    tables, the zero bias) and their ``total``; ``build_peak`` adds the NF4 load's staging chunk.  The KV cache and the
    activations grow with the calls and are not counted."""
    H, F, L, V = cfg.hidden, cfg.ffn, cfg.layers, cfg.vocab_size
    QD, KD = cfg.heads * cfg.head_dim, cfg.kv_heads * cfg.head_dim
    shapes = [(QD + 2 * KD, H), (H, QD), (2 * F, H), (H, F)]
    n = sum(a * b for a, b in shapes)
    nf4 = weights == "nf4"
    plan = {
        "layers": L * (n // 2 + n // 64 * 4) if nf4 else L * n * 4,
        "embeddings": V * H * 4,
        "lm_head": V * H * 4 + V * 4,
        "scratch": 4 * max(a * b for a, b in shapes) if nf4 else 0,
        "other": 4 * (L * (2 * H + (2 * cfg.head_dim if isinstance(cfg, Qwen3Config) else 0)) + H
                      + 2 * cfg.max_pos * cfg.head_dim // 2 + max(QD + 2 * KD, 2 * F, H)),
    }
    plan["total"] = sum(plan.values())
    plan["build_peak"] = plan["total"] + (NF4_LOAD_STAGING if nf4 else 0)
    return plan


def check_decoder_plan(cfg: BertConfig, weights: str, free_bytes: Optional[int] = None) -> Dict[str, int]:
    """``decoder_memory_plan``, refused with a ValueError naming the bytes and the setting: split weights above hidden
    4096 (NF4 takes them), and, given the device's free bytes, a plan that does not fit"""
    plan = decoder_memory_plan(cfg, weights)
    name = getattr(cfg, "name", "decoder")
    if weights != "nf4" and cfg.hidden > SPLIT_MAX_HIDDEN:
        raise ValueError(
            f"{name}: hidden_size {cfg.hidden} > {SPLIT_MAX_HIDDEN} runs on NF4 weights only; split planes would need "
            f"{plan['layers'] / GB:.1f} GB for the layers ({plan['total']} bytes in all): set RMU_DECODER_WEIGHTS=nf4, "
            f"which plans {decoder_memory_plan(cfg, 'nf4')['total'] / GB:.1f} GB")
    if free_bytes is not None and plan["build_peak"] > free_bytes:
        raise ValueError(
            f"{name}: the decoder needs {plan['build_peak']} bytes ({plan['build_peak'] / GB:.1f} GB) of device memory "
            f"with RMU_DECODER_WEIGHTS={weights}, and the device has {free_bytes} bytes ({free_bytes / GB:.1f} GB) free"
            + ("; RMU_DECODER_WEIGHTS=nf4 plans " f"{decoder_memory_plan(cfg, 'nf4')['build_peak'] / GB:.1f} GB"
               if weights != "nf4" else ""))
    return plan


def decoder_lm_head(model_name: str, cfg: BertConfig, cache_folder: Optional[str] = None) -> np.ndarray:
    """the decoder's LM head [vocab_size, H] float32: ``lm_head.weight``, or ``embed_tokens`` when config.json sets
    ``tie_word_embeddings`` (or the snapshot has no lm_head); for ``synthetic:<preset>[:seed[:scale]]`` seeded rows
    N(0, 0.02 scale) drawn after the decoder's weights"""
    if model_name.startswith("synthetic:"):
        parts = model_name.split(":")
        seed = int(parts[2]) if len(parts) > 2 else 0
        scale = float(parts[3]) if len(parts) > 3 else 1.0
        rng = np.random.default_rng([seed, 1])
        return np.ascontiguousarray(0.02 * scale * rng.standard_normal((cfg.vocab_size, cfg.hidden)), dtype=np.float32)
    path = find_snapshot(model_name, cache_folder)
    tied = bool((_read_json(os.path.join(path, "config.json")) or {}).get("tie_word_embeddings", False))
    names = ([] if tied else ["lm_head.weight"]) + ["model.embed_tokens.weight", "embed_tokens.weight"]
    for name in names:
        w = _load_tensors(path, lambda n, name=name: n == name)
        if name in w:
            return np.ascontiguousarray(w[name], dtype=np.float32)
    raise KeyError(f"{path}: no lm_head.weight or embed_tokens.weight")


def find_snapshot(model_name: str, cache_folder: Optional[str] = None) -> str:
    """the local snapshot directory of a model id: the id itself, or ``<cache>/<name>`` / ``$RAGMEUP_MODEL_DIR/<name>``
    (each also with the id's last path component)"""
    cands = [model_name]
    for root in (cache_folder, os.environ.get("RAGMEUP_MODEL_DIR")):
        if root:
            cands += [os.path.join(root, model_name), os.path.join(root, model_name.split("/")[-1])]
    for c in cands:
        if os.path.isdir(c):
            return c
    raise FileNotFoundError(
        f"model {model_name!r} not found locally (no network in this deployment): point "
        f"RAGMEUP_MODEL_DIR at a directory holding its HuggingFace snapshot, or use 'synthetic:<preset>'")


REL_EMB = "encoder.rel_embeddings.weight"
REL_LN = ("encoder.LayerNorm.weight", "encoder.LayerNorm.bias")


def deberta_to_canonical(raw: Dict[str, np.ndarray], cfg: DebertaConfig) -> Dict[str, np.ndarray]:
    """DeBERTa-v2 tensors (bare, or under ``deberta.`` as the sequence-classification model saves them) -> the
    canonical names of ``weight_names``: ``query_proj`` / ``key_proj`` / ``value_proj`` -> ``query`` / ``key`` /
    ``value``, zero position and token-type tables, rows 0..2s of ``rel_embeddings``; ``pooler.dense`` and
    ``classifier`` keep their names."""
    w: Dict[str, np.ndarray] = {}
    for k, v in raw.items():
        k = k[8:] if k.startswith("deberta.") else k
        for a in ("query", "key", "value"):
            k = k.replace(f"attention.self.{a}_proj.", f"attention.self.{a}.")
        w[k] = np.ascontiguousarray(v, dtype=np.float32)
    w["embeddings.position_embeddings.weight"] = np.zeros((cfg.max_pos, cfg.hidden), np.float32)
    w["embeddings.token_type_embeddings.weight"] = np.zeros((1, cfg.hidden), np.float32)
    if REL_EMB in w:
        w[REL_EMB] = np.ascontiguousarray(w[REL_EMB][:2 * cfg.position_buckets])
    return w


def adapter_prefix(layer: int, language: str) -> str:
    return f"encoder.layer.{layer}.output.adapter_modules.{language}."


# config.json model_type -> how the snapshot is read; a config without model_type is read as BERT
MODEL_TYPES = ("bert", "mpnet", "roberta", "xlm-roberta", "xmod", "deberta-v2", "modernbert", "qwen3", "distilbert")


# shapes of the models BASELINE.json / .env.template name (SURVEY.md §2.2 table)
PRESETS: Dict[str, Tuple[BertConfig, str, int]] = {
    # name: (config, pooling, max_seq_length)
    "all-MiniLM-L6-v2": (BertConfig(hidden=384, layers=6, heads=12, ffn=1536), "mean", 256),
    "ms-marco-MiniLM-L-6-v2": (BertConfig(hidden=384, layers=6, heads=12, ffn=1536, num_labels=1), "cls", 512),
    "bge-base-en-v1.5": (BertConfig(hidden=768, layers=12, heads=12, ffn=3072), "cls", 512),
    "GIST-small-Embedding-v0": (BertConfig(hidden=384, layers=12, heads=12, ffn=1536), "cls", 512),
    # tiny shapes for unit tests
    "tiny": (BertConfig(vocab_size=1000, hidden=128, layers=2, heads=4, ffn=256, max_pos=128), "mean", 64),
    # the BERT rerankers FlashRank ships (FLASHRANK_MODELS)
    "ms-marco-MultiBERT-L-12": (BertConfig(vocab_size=105879, hidden=768, layers=12, heads=12, ffn=3072, num_labels=2),
                                "cls", 512),
    "ms-marco-TinyBERT-L-2-v2": (BertConfig(hidden=128, layers=2, heads=2, ffn=512, num_labels=1), "cls", 512),
    "ms-marco-MiniLM-L-12-v2": (BertConfig(hidden=384, layers=12, heads=12, ffn=1536, num_labels=1), "cls", 512),
    # MPNet sentence embedders (HuggingFaceEmbeddings' default model; Normalize follows the preset's own pipeline)
    "all-mpnet-base-v2": (MPNetConfig(hidden=768, layers=12, heads=12, ffn=3072), "mean", 384),
    "multi-qa-mpnet-base-dot-v1": (MPNetConfig(hidden=768, layers=12, heads=12, ffn=3072), "cls", 512),
    "tiny-mpnet": (MPNetConfig(vocab_size=1000, hidden=128, layers=2, heads=4, ffn=256, max_pos=130), "mean", 64),
    # XLM-R: the bge rerankers (HuggingFaceCrossEncoder's default model) and the multilingual embedders
    "bge-reranker-base": (XLMRConfig(hidden=768, layers=12, heads=12, ffn=3072), "cls", 512),
    "bge-reranker-v2-m3": (XLMRConfig(hidden=1024, layers=24, heads=16, ffn=4096, max_pos=8194), "cls", 8192),
    "multilingual-e5-small": (XLMRConfig(vocab_size=250037, hidden=384, layers=12, heads=12, ffn=1536), "mean", 512),
    "multilingual-e5-base": (XLMRConfig(hidden=768, layers=12, heads=12, ffn=3072), "mean", 512),
    "bge-m3": (XLMRConfig(hidden=1024, layers=24, heads=16, ffn=4096, max_pos=8194), "cls", 8192),
    "paraphrase-multilingual-mpnet-base-v2": (XLMRConfig(hidden=768, layers=12, heads=12, ffn=3072), "mean", 128),
    "tiny-xlmr": (XLMRConfig(vocab_size=2000, hidden=128, layers=2, heads=4, ffn=256, max_pos=130), "mean", 64),
    "tiny-xlmr-long": (XLMRConfig(vocab_size=2000, hidden=128, layers=2, heads=4, ffn=256, max_pos=8194), "cls", 8192),
    # X-MOD: XLM-R base with one adapter per language (adapter_reduction_factor 2); the preset's language is its default
    "xmod-base": (XmodConfig(hidden=768, layers=12, heads=12, ffn=3072, adapter_dim=384), "mean", 512),
    "tiny-xmod": (XmodConfig(vocab_size=2000, hidden=256, layers=2, heads=4, ffn=512, max_pos=130, adapter_dim=128),
                  "mean", 64),
    # DeBERTa-v3 rerankers (mixedbread-ai/mxbai-rerank-*-v1): position_buckets 256, max_position_embeddings 512
    "mxbai-rerank-xsmall-v1": (DebertaConfig(hidden=384, layers=12, heads=6, ffn=1536), "cls", 512),
    "mxbai-rerank-base-v1": (DebertaConfig(hidden=768, layers=12, heads=12, ffn=3072), "cls", 512),
    "mxbai-rerank-large-v1": (DebertaConfig(hidden=1024, layers=24, heads=16, ffn=4096), "cls", 512),
    "tiny-deberta": (DebertaConfig(vocab_size=2000, hidden=128, layers=2, heads=2, ffn=256), "cls", 512),
    # ModernBERT: the base and large shapes of the published configs [3P-recall: not checkable here]; the reranker
    # pools by CLS (the base model's classifier_pooling default), modernbert-embed by mean + Normalize, gte-modernbert
    # by CLS.  A snapshot's config.json and sentence-transformers modules override all of this.
    "modernbert-base": (ModernBertConfig(hidden=768, layers=22, heads=12, ffn=1152), "cls", 8192),
    "modernbert-large": (ModernBertConfig(hidden=1024, layers=28, heads=16, ffn=2624), "cls", 8192),
    "gte-reranker-modernbert-base": (ModernBertConfig(hidden=768, layers=22, heads=12, ffn=1152), "cls", 8192),
    "modernbert-embed-base": (ModernBertConfig(hidden=768, layers=22, heads=12, ffn=1152, classifier_pooling="mean"),
                              "mean", 8192),
    "gte-modernbert-base": (ModernBertConfig(hidden=768, layers=22, heads=12, ffn=1152), "cls", 8192),
    # four layers, so both layer types and layer 0's identity attn_norm appear; and a small window (|i - j| <= 16), so
    # short sequences cross many window blocks
    "tiny-modernbert": (ModernBertConfig(vocab_size=1000, hidden=128, layers=4, heads=2, ffn=192, max_pos=1024),
                        "mean", 1024),
    "tiny-modernbert-window": (ModernBertConfig(vocab_size=1000, hidden=128, layers=4, heads=2, ffn=192, max_pos=1024,
                                                layer_windows=modernbert_windows(4, 3, 32), classifier_pooling="mean"),
                               "mean", 1024),
    # Qwen3: the 0.6B shape of Qwen3-Embedding-0.6B and Qwen3-Reranker-0.6B [3P-recall: their config.json is not read
    # here]; pooling "last" is the last-token row.  tiny-qwen3: head_dim 128, two query heads per kv head, three layers.
    "qwen3-embedding-0.6b": (Qwen3Config(), "last", 8192),
    "qwen3-reranker-0.6b": (Qwen3Config(reranker=True, num_labels=2), "last", 8192),
    "tiny-qwen3": (Qwen3Config(vocab_size=1000, hidden=256, layers=3, heads=4, ffn=384, max_pos=8192, kv_heads=2,
                               rope_theta=10000.0, tie_word_embeddings=False, pad_token_id=0), "last", 8192),
    # sentence-transformers models with a Dense module after pooling (DENSE_PRESETS) [3P-recall: their config.json and
    # module files are not read here].  distiluse-base-multilingual-cased-v2: DistilBERT, mean pooling, Dense 768 -> 512
    # tanh, no Normalize.  LaBSE: BERT, CLS pooling, Dense 768 -> 768 tanh, Normalize.  tiny-distilbert: a widening
    # Dense, so the output is wider than hidden.
    "distiluse-base-multilingual-cased-v2": (DistilBertConfig(vocab_size=119547), "mean", 128),
    "LaBSE": (BertConfig(vocab_size=501153, hidden=768, layers=12, heads=12, ffn=3072), "cls", 256),
    "tiny-distilbert": (DistilBertConfig(vocab_size=1000, hidden=128, layers=2, heads=4, ffn=256, max_pos=128), "mean", 64),
}

# presets whose sentence-transformers pipeline has no Normalize module
UNNORMALIZED_PRESETS = {"multi-qa-mpnet-base-dot-v1", "paraphrase-multilingual-mpnet-base-v2", "gte-modernbert-base",
                        "distiluse-base-multilingual-cased-v2", "tiny-distilbert"}

# Dense modules of the presets above, in order: (out_features, bias, activation)
DENSE_PRESETS: Dict[str, Tuple[Tuple[int, bool, str], ...]] = {
    "distiluse-base-multilingual-cased-v2": ((512, True, "tanh"),),
    "LaBSE": ((768, True, "tanh"),),
    "tiny-distilbert": ((200, True, "tanh"),),
}

# FlashRank's model names -> the public HuggingFace checkpoints its ONNX files were exported from [3P-recall: flashrank
# 0.2.x; the mapping is recalled, not read, and is unverified].  Only the BERT cross-encoders are here: FlashRank's T5
# (rank-T5-flan) and listwise LLM (rank_zephyr_7b_v1_full) models are not BERT encoders.
FLASHRANK_MODELS: Dict[str, str] = {
    "ms-marco-MultiBERT-L-12": "amberoad/bert-multilingual-passage-reranking-msmarco",
    "ms-marco-TinyBERT-L-2-v2": "cross-encoder/ms-marco-TinyBERT-L-2-v2",
    "ms-marco-MiniLM-L-12-v2": "cross-encoder/ms-marco-MiniLM-L-12-v2",
}


def weight_names(cfg: BertConfig, with_head: bool):
    if isinstance(cfg, LlamaConfig):
        return llama_weight_names(cfg)
    if isinstance(cfg, Qwen3Config):
        return qwen3_weight_names(cfg, with_head)
    if isinstance(cfg, ModernBertConfig):
        return modernbert_weight_names(cfg, with_head)
    H, F = cfg.hidden, cfg.ffn
    names = [
        ("embeddings.word_embeddings.weight", (cfg.vocab_size, H)),
        ("embeddings.position_embeddings.weight", (cfg.max_pos, H)),
        ("embeddings.token_type_embeddings.weight", (cfg.type_vocab, H)),
        ("embeddings.LayerNorm.weight", (H,)),
        ("embeddings.LayerNorm.bias", (H,)),
    ]
    for l in range(cfg.layers):
        p = f"encoder.layer.{l}."
        names += [
            (p + "attention.self.query.weight", (H, H)), (p + "attention.self.query.bias", (H,)),
            (p + "attention.self.key.weight", (H, H)), (p + "attention.self.key.bias", (H,)),
            (p + "attention.self.value.weight", (H, H)), (p + "attention.self.value.bias", (H,)),
            (p + "attention.output.dense.weight", (H, H)), (p + "attention.output.dense.bias", (H,)),
            (p + "attention.output.LayerNorm.weight", (H,)), (p + "attention.output.LayerNorm.bias", (H,)),
            (p + "intermediate.dense.weight", (F, H)), (p + "intermediate.dense.bias", (F,)),
            (p + "output.dense.weight", (H, F)), (p + "output.dense.bias", (H,)),
            (p + "output.LayerNorm.weight", (H,)), (p + "output.LayerNorm.bias", (H,)),
        ]
    if with_head:
        names += [
            ("pooler.dense.weight", (H, H)), ("pooler.dense.bias", (H,)),
            ("classifier.weight", (cfg.num_labels, H)), ("classifier.bias", (cfg.num_labels,)),
        ]
    if cfg.rel_buckets:
        names.append((REL_BIAS, (cfg.rel_buckets, cfg.heads)))
    if cfg.adapter_dim:
        for l in range(cfg.layers):
            names += adapter_names(cfg, l, cfg.language)
    if cfg.position_buckets:
        names += [(REL_EMB, (2 * cfg.position_buckets, H)), (REL_LN[0], (H,)), (REL_LN[1], (H,))]
    return names


def adapter_names(cfg: BertConfig, layer: int, language: str):
    """the four tensors of one X-MOD adapter, in the order rmu_encoder_create takes them"""
    H, A = cfg.hidden, cfg.adapter_dim
    p = adapter_prefix(layer, language)
    return [(p + "dense1.weight", (A, H)), (p + "dense1.bias", (A,)), (p + "dense2.weight", (H, A)),
            (p + "dense2.bias", (H,))]


REL_BIAS = "encoder.relative_attention_bias.weight"
# MPNet checkpoint names -> the BERT names above (the embeddings and the FFN blocks have BERT's names already)
_MPNET_RENAME = (("attention.attn.q.", "attention.self.query."), ("attention.attn.k.", "attention.self.key."),
                 ("attention.attn.v.", "attention.self.value."), ("attention.attn.o.", "attention.output.dense."),
                 ("attention.LayerNorm.", "attention.output.LayerNorm."))


def mpnet_to_canonical(raw: Dict[str, np.ndarray], cfg: MPNetConfig) -> Dict[str, np.ndarray]:
    """MPNet tensors (bare or under ``mpnet.``) -> the canonical names of ``weight_names``: q/k/v/o and the attention
    LayerNorm renamed, a zero [1, H] token-type table, and rows 0..31 of the relative bias (transformers looks up 32
    buckets whatever the table holds)."""
    w: Dict[str, np.ndarray] = {}
    for k, v in raw.items():
        k = k[6:] if k.startswith("mpnet.") else k
        for a, b in _MPNET_RENAME:
            k = k.replace(a, b)
        w[k] = np.ascontiguousarray(v, dtype=np.float32)
    w["embeddings.token_type_embeddings.weight"] = np.zeros((1, cfg.hidden), np.float32)
    if REL_BIAS in w:
        w[REL_BIAS] = np.ascontiguousarray(w[REL_BIAS][:cfg.rel_buckets])
    return w


def xlmr_to_canonical(raw: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """XLM-R / RoBERTa tensors (bare, as ``XLMRobertaModel.save_pretrained`` writes them, or under ``roberta.``, as the
    sequence-classification model does) -> the canonical names of ``weight_names``.  The classification head's
    ``classifier.dense`` is the pooler and ``classifier.out_proj`` the classifier; a bare ``pooler.*`` (the embedder's
    unused BertPooler) is dropped, so it never stands in for a head."""
    w: Dict[str, np.ndarray] = {}
    for k, v in raw.items():
        if k.startswith("pooler."):
            continue
        k = k[8:] if k.startswith("roberta.") else k
        if k.startswith("classifier.dense."):
            k = "pooler.dense." + k[17:]
        elif k.startswith("classifier.out_proj."):
            k = "classifier." + k[20:]
        w[k] = np.ascontiguousarray(v, dtype=np.float32)
    return w


def synthetic_bert_weights(cfg: BertConfig, seed: int = 0, with_head: bool = False,
                           scale: float = 1.0) -> Dict[str, np.ndarray]:
    """Seeded random weights.  ``scale=1`` is BERT's init (N(0, 0.02)) with small
    random biases and LayerNorm gains near 1; ``scale>1`` widens the linear
    weights to a "trained-like" regime (saturating softmax, logits of order 10).  An X-MOD config gets an adapter set for
    every one of its languages, drawn after the rest from a second stream, so the other tensors are those of the XLM-R
    config of the same shape and seed."""
    rng = np.random.default_rng(seed)
    out: Dict[str, np.ndarray] = {}
    names = [(n, s, rng) for n, s in weight_names(cfg, with_head) if ".adapter_modules." not in n]
    if cfg.adapter_dim:
        rng2 = np.random.default_rng(seed + 104729)
        names += [(n, s, rng2) for lang in cfg.languages for l in range(cfg.layers) for n, s in adapter_names(cfg, l, lang)]
    for name, shape, rng in names:
        if isinstance(cfg, ModernBertConfig) and (name.endswith(".bias") or name.startswith("layers.0.attn_norm.")):
            # ModernBERT has no biases or LayerNorm shifts (attention_bias, mlp_bias, norm_bias false), and no attn_norm
            # in layer 0
            a = np.ones(shape) if name == "layers.0.attn_norm.weight" else np.zeros(shape)
        elif isinstance(cfg, ModernBertConfig) and name.endswith("norm.weight"):
            a = 1.0 + 0.1 * rng.standard_normal(shape)
        elif isinstance(cfg, ModernBertConfig) and name.startswith("embeddings."):
            a = 0.02 * rng.standard_normal(shape) * (3.0 if scale > 1 else 1.0)
        elif name == REL_BIAS:                     # a few units across buckets, as trained MPNet biases spread
            a = rng.standard_normal(shape)
        elif name == "embeddings.token_type_embeddings.weight" and isinstance(cfg, (MPNetConfig, DebertaConfig,
                                                                                   DistilBertConfig)):
            a = np.zeros(shape)                    # MPNet, DeBERTa and DistilBERT have no token types (XLM-R's one row is trained)
        elif name == "embeddings.position_embeddings.weight" and isinstance(cfg, DebertaConfig):
            a = np.zeros(shape)                    # nor absolute positions (position_biased_input false)
        elif name.endswith("LayerNorm.weight"):
            a = 1.0 + 0.1 * rng.standard_normal(shape)
        elif name.endswith("LayerNorm.bias"):
            a = 0.05 * rng.standard_normal(shape)
        elif name.endswith(".bias"):
            a = 0.02 * scale * rng.standard_normal(shape)
        elif name.startswith("embeddings."):
            a = 0.02 * rng.standard_normal(shape) * (3.0 if scale > 1 else 1.0)
        else:
            a = 0.02 * scale * rng.standard_normal(shape)
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    return out


# sentence-transformers Dense activations -> RMU_DENSE_IDENTITY / RMU_DENSE_TANH
DENSE_ACTIVATIONS = {"identity": 0, "tanh": 1}
_DENSE_CLASSES = {"torch.nn.modules.linear.Identity": "identity", "torch.nn.modules.activation.Tanh": "tanh"}
MODULE_KINDS = ("Transformer", "Pooling", "Dense", "Normalize")


def dense_layers(w: Dict[str, np.ndarray]):
    """the Dense chain a weight dict holds, in order: [(weight [out, in], bias [out] or None, RMU_DENSE_* code)], from
    ``dense.<i>.weight``, ``dense.<i>.bias`` (absent without a bias) and ``dense.<i>.activation`` (a 0-d int32 code)"""
    out = []
    while f"dense.{len(out)}.weight" in w:
        i = len(out)
        out.append((w[f"dense.{i}.weight"], w.get(f"dense.{i}.bias"), int(w[f"dense.{i}.activation"])))
    return out


def synthetic_dense_weights(hidden: int, layers, seed: int = 0, scale: float = 1.0) -> Dict[str, np.ndarray]:
    """seeded Dense modules of DENSE_PRESETS' form, N(0, 0.02 scale) weights and biases, from a stream of their own (the
    encoder's weights are those of the same preset without Dense)"""
    rng = np.random.default_rng(seed + 15485863)
    w: Dict[str, np.ndarray] = {}
    d_in = hidden
    for i, (d_out, bias, act) in enumerate(layers):
        w[f"dense.{i}.weight"] = (0.02 * scale * rng.standard_normal((d_out, d_in))).astype(np.float32)
        if bias:
            w[f"dense.{i}.bias"] = (0.02 * scale * rng.standard_normal(d_out)).astype(np.float32)
        w[f"dense.{i}.activation"] = np.array(DENSE_ACTIVATIONS[act], np.int32)
        d_in = d_out
    return w


def module_entries(path: str):
    """modules.json of a sentence-transformers snapshot -> [(kind, module dir)] in order; a module type other than
    Transformer, Pooling, Dense or Normalize is refused with a ValueError naming the module (the encoder would return a
    vector that module never saw)"""
    entries = []
    for m in _read_json(os.path.join(path, "modules.json")) or []:
        t = m.get("type", "")
        kind = t.rsplit(".", 1)[-1]
        if kind not in MODULE_KINDS:
            raise ValueError(f"{path}: sentence-transformers module {m.get('path') or m.get('name')!r} of type {t!r} is "
                             f"not supported: the encoder computes {', '.join(MODULE_KINDS)} modules only")
        entries.append((kind, m.get("path", "")))
    return entries


def read_modules(path: str, hidden: int):
    """``module_entries`` and the Dense weights in the form of ``dense_layers``.  Refused with a ValueError naming the
    module or field: a Dense before Pooling or a Normalize before a Dense (sentence-transformers runs Pooling ->
    Dense... -> Normalize); a Dense activation other than Tanh or Identity; in_features that do not chain from hidden;
    a weight or bias that does not match its config."""
    entries = module_entries(path)
    kinds = [k for k, _ in entries]
    w: Dict[str, np.ndarray] = {}
    d_in, i = hidden, 0
    for pos, (kind, mdir) in enumerate(entries):
        if kind != "Dense":
            continue
        if "Pooling" not in kinds[:pos]:
            raise ValueError(f"{path}: Dense module {mdir!r} comes before Pooling; the encoder runs Pooling -> Dense")
        if "Normalize" in kinds[:pos]:
            raise ValueError(f"{path}: Normalize comes before Dense module {mdir!r}; the encoder runs Dense -> Normalize")
        dc = _read_json(os.path.join(path, mdir, "config.json")) or {}
        act = _DENSE_CLASSES.get(dc.get("activation_function", "torch.nn.modules.activation.Tanh"))
        if act is None:
            raise ValueError(f"{path}: Dense module {mdir!r} with activation_function = {dc['activation_function']!r} is "
                             f"not supported: Tanh and Identity are computed")
        if int(dc.get("in_features", -1)) != d_in:
            raise ValueError(f"{path}: Dense module {mdir!r} with in_features = {dc.get('in_features')!r} does not chain: "
                             f"its input is {d_in} wide")
        d_out, bias = int(dc.get("out_features", 0)), bool(dc.get("bias", True))
        t = _load_tensors(os.path.join(path, mdir))
        W, b = t.get("linear.weight"), t.get("linear.bias")
        if W is None or W.shape != (d_out, d_in) or (b is not None) != bias or (bias and b.shape != (d_out,)):
            raise ValueError(f"{path}: Dense module {mdir!r}: linear.weight {None if W is None else W.shape} / linear.bias "
                             f"{None if b is None else b.shape} do not match out_features = {d_out}, in_features = "
                             f"{d_in}, bias = {bias}")
        w[f"dense.{i}.weight"] = np.ascontiguousarray(W, dtype=np.float32)
        if bias:
            w[f"dense.{i}.bias"] = np.ascontiguousarray(b, dtype=np.float32)
        w[f"dense.{i}.activation"] = np.array(DENSE_ACTIVATIONS[act], np.int32)
        d_in, i = d_out, i + 1
    return entries, w


def _read_json(path: str) -> Optional[dict]:
    if os.path.exists(path):
        with open(path) as f:
            return json.load(f)
    return None


def _load_tensors(path: str, keep=None) -> Dict[str, np.ndarray]:
    """``model.safetensors``, or for snapshots that ship only the older format (the multilingual MS MARCO reranker
    behind FlashRank's default) ``pytorch_model.bin``, read with ``weights_only=True`` so no pickled code runs.
    ``keep(name)`` (optional) selects tensors: from safetensors only those are read; a pickle is read whole and
    filtered."""
    st = os.path.join(path, "model.safetensors")
    pt = os.path.join(path, "pytorch_model.bin")
    if not os.path.exists(st) and os.path.exists(pt):
        import torch
        sd = torch.load(pt, weights_only=True, map_location="cpu")
        return {k: v.detach().to(torch.float32).numpy() for k, v in sd.items()
                if v.is_floating_point() and (keep is None or keep(k))}
    if not os.path.exists(st) and os.path.exists(os.path.join(path, SHARD_INDEX)):
        out: Dict[str, np.ndarray] = {}
        for f in _safetensors_files(path):
            out.update(_load_safetensors(f, keep))
        return out
    return _load_safetensors(st, keep)


SHARD_INDEX = "model.safetensors.index.json"


def _safetensors_files(path: str):
    """``model.safetensors``, or the shards ``model.safetensors.index.json`` lists, in its order"""
    st = os.path.join(path, "model.safetensors")
    idx = _read_json(os.path.join(path, SHARD_INDEX))
    if os.path.exists(st) or idx is None:
        return [st]
    return [os.path.join(path, f) for f in dict.fromkeys(idx["weight_map"].values())]


def _load_safetensors(st: str, keep=None) -> Dict[str, np.ndarray]:
    """one safetensors file (all tensors, or those ``keep`` selects) read by numpy; a file numpy cannot read (bfloat16,
    which numpy has no type for) is read through torch instead, its bfloat16 tensors widened to float32 (exact)"""
    from safetensors import safe_open
    try:
        if keep is None:
            from safetensors.numpy import load_file
            return load_file(st)
        with safe_open(st, framework="numpy") as f:
            return {k: f.get_tensor(k) for k in f.keys() if keep(k)}
    except TypeError:
        import torch
        with safe_open(st, framework="pt") as f:
            return {k: (t.to(torch.float32) if t.dtype == torch.bfloat16 else t).numpy()
                    for k in f.keys() if keep is None or keep(k) for t in (f.get_tensor(k),)}


def _xmod_keep(language: str):
    """tensor filter of an X-MOD snapshot: everything but the adapters of the other languages"""
    mine = f".adapter_modules.{language}."
    return lambda name: ".adapter_modules." not in name or mine in name


def load_hf_snapshot(path: str, with_head: bool):
    """Read a local HF / sentence-transformers snapshot.  Returns
    (config, weights, pooling, normalize, max_seq_length, activation)."""
    cfgd = _read_json(os.path.join(path, "config.json"))
    if cfgd is None:
        raise FileNotFoundError(f"{path}: no config.json")
    kind = cfgd.get("model_type", "bert")
    if kind not in MODEL_TYPES:
        raise ValueError(f"{path}: model_type {kind!r} is not supported; the encoder runs {', '.join(MODEL_TYPES)}")
    if kind == "qwen3":
        return _load_qwen3_snapshot(path, cfgd, with_head)
    mpnet, xlmr, deberta = kind == "mpnet", kind in ("roberta", "xlm-roberta", "xmod"), kind == "deberta-v2"
    modern, distil = kind == "modernbert", kind == "distilbert"
    if mpnet and with_head:
        raise ValueError(f"{path}: MPNet cross-encoders are not supported (MPNet runs as a sentence embedder only)")
    if deberta and not with_head:
        raise ValueError(f"{path}: model_type 'deberta-v2' runs as a cross-encoder (reranker) only, not as an embedder")
    if kind == "xmod":
        cfg = XmodConfig.from_hf(cfgd, path)
    elif modern:
        cfg = ModernBertConfig.from_hf(cfgd)
    elif deberta:
        cfg = DebertaConfig.from_hf(cfgd)
    elif distil:
        cfg = DistilBertConfig.from_hf(cfgd)
    else:
        cfg = MPNetConfig.from_hf(cfgd) if mpnet else XLMRConfig.from_hf(cfgd) if xlmr else BertConfig.from_hf(cfgd)
    raw = _load_tensors(path, _xmod_keep(cfg.language) if cfg.adapter_dim else None)
    if mpnet:
        w = mpnet_to_canonical(raw, cfg)
    elif modern:
        w = modernbert_to_canonical(raw, cfg, with_head)
    elif deberta:
        w = deberta_to_canonical(raw, cfg)
    elif xlmr:
        w = xlmr_to_canonical(raw)
    elif distil:
        w = distilbert_to_canonical(raw, cfg)
    else:
        w: Dict[str, np.ndarray] = {}
        for k, v in raw.items():
            k2 = k[5:] if k.startswith("bert.") else k
            w[k2] = np.ascontiguousarray(v, dtype=np.float32)
    need = [n for n, _ in weight_names(cfg, with_head)]
    missing = [n for n in need if n not in w]
    if missing:
        raise KeyError(f"{path}: missing tensors {missing[:4]}...")
    pooling, normalize, max_len = "mean", False, min(cfg.max_pos - cfg.position_offset, 512)
    if modern:
        # sequences up to max_position_embeddings, within the tokenizer's model_max_length
        max_len = cfg.max_pos
        tc = _read_json(os.path.join(path, "tokenizer_config.json")) or {}
        if tc.get("model_max_length") is not None:
            max_len = min(int(tc["model_max_length"]), max_len)
    if deberta:
        # CrossEncoder passes max_length=None: the tokenizer's model_max_length, within max_position_embeddings
        max_len = cfg.max_pos
        tc = _read_json(os.path.join(path, "tokenizer_config.json")) or {}
        if tc.get("model_max_length") is not None:
            max_len = min(int(tc["model_max_length"]), max_len)
    if xlmr:
        # CrossEncoder passes max_length=None, so the tokenizer's model_max_length applies [3P-recall]; positions end
        # at max_pos - 2 tokens either way (8192 for bge-m3 and bge-reranker-v2-m3)
        max_len = cfg.max_pos - cfg.position_offset
        tc = _read_json(os.path.join(path, "tokenizer_config.json")) or {}
        if tc.get("model_max_length") is not None:
            max_len = min(int(tc["model_max_length"]), max_len)
    mods, dense = read_modules(path, cfg.hidden)
    w.update(dense)
    for kind, mdir in mods:
        if kind == "Pooling":
            pc = _read_json(os.path.join(path, mdir, "config.json")) or {}
            if pc.get("pooling_mode_cls_token"):
                pooling = "cls"
            elif pc.get("pooling_mode_mean_tokens", True):
                pooling = "mean"
            else:
                raise ValueError("unsupported pooling mode in " + mdir)
        if kind == "Normalize":
            normalize = True
    sb = _read_json(os.path.join(path, "sentence_bert_config.json"))
    if sb and sb.get("max_seq_length"):
        max_len = int(sb["max_seq_length"])
    act = "identity"
    a = cfgd.get("sbert_ce_default_activation_function")
    if with_head:
        if a is None:
            act = "sigmoid" if cfg.num_labels == 1 else "identity"
        else:
            act = "sigmoid" if "Sigmoid" in a else "identity"
    return cfg, w, pooling, normalize, max_len, act


# Qwen3-Reranker's prompt, from its model card [3P-recall: the card is not readable here]: the chat prefix with the
# judging instruction, the suffix that opens an empty <think> block, and the default task instruction.  The score is
# P(yes) = exp(log_softmax([logit("no"), logit("yes")])[1]) at the last token.
QWEN3_RERANK_PREFIX = ("<|im_start|>system\nJudge whether the Document meets the requirements based on the Query and the "
                       "Instruct provided. Note that the answer can only be \"yes\" or \"no\".<|im_end|>\n"
                       "<|im_start|>user\n")
QWEN3_RERANK_SUFFIX = "<|im_end|>\n<|im_start|>assistant\n<think>\n\n</think>\n\n"
QWEN3_RERANK_INSTRUCTION = "Given a web search query, retrieve relevant passages that answer the query"
QWEN3_RERANK_MAX_LENGTH = 8192      # the model card's max_length [3P-recall]


def _load_qwen3_snapshot(path: str, cfgd: dict, with_head: bool):
    """a ``qwen3`` snapshot -> (config, weights, pooling, normalize, max_len, activation).  Embedders (no head) pool by
    the last token; ``1_Pooling`` must say ``pooling_mode_lasttoken``.  With a head: ``Qwen3ForSequenceClassification``
    (``score.weight``, needs ``pad_token_id``), or a causal LM (``Qwen3ForCausalLM``, Qwen3-Reranker), which scores
    P(yes) from the [no, yes] rows of ``lm_head`` (activation ``"yes_prob"``)."""
    if not os.path.exists(os.path.join(path, "tokenizer.json")):
        raise ValueError(f"{path}: a qwen3 snapshot needs tokenizer.json (its byte-level BPE has no other file form here)")
    cfg = Qwen3Config.from_hf(cfgd, name=path)
    archs = cfgd.get("architectures") or []
    names = set().union(*[_tensor_names_file(f) for f in _safetensors_files(path)])
    seqcls = "score.weight" in names or "Qwen3ForSequenceClassification" in archs
    keep = (lambda n: n not in ("lm_head.weight", "score.weight")) if not with_head else (lambda n: n != "lm_head.weight")
    w = qwen3_to_canonical(_load_tensors(path, keep), cfg)
    act = "identity"
    if with_head and seqcls:
        if cfg.pad_token_id is None:
            raise ValueError(f"{path}: a Qwen3ForSequenceClassification snapshot needs pad_token_id: its head reads the "
                             f"rightmost token that is not padding (transformers refuses batches without it)")
        cfg.num_labels = int(w["head"].shape[0])
        a = cfgd.get("sbert_ce_default_activation_function")
        act = ("sigmoid" if cfg.num_labels == 1 else "identity") if a is None else ("sigmoid" if "Sigmoid" in a else "identity")
    elif with_head:
        from tokenizers import Tokenizer
        tok = Tokenizer.from_file(os.path.join(path, "tokenizer.json"))
        yes, no = tok.token_to_id("yes"), tok.token_to_id("no")
        if yes is None or no is None:
            raise ValueError(f"{path}: the reranker's tokenizer has no single 'yes' / 'no' tokens to score with")
        cfg.reranker, cfg.num_labels = True, 2
        w["head"] = qwen3_lm_rows(path, cfg, [no, yes])
        act = "yes_prob"
    missing = [n for n, _ in qwen3_weight_names(cfg, with_head) if n not in w]
    if missing:
        raise KeyError(f"{path}: missing tensors {missing[:4]}...")
    tc = _read_json(os.path.join(path, "tokenizer_config.json")) or {}
    max_len = cfg.max_pos
    if cfg.reranker:
        max_len = min(max_len, QWEN3_RERANK_MAX_LENGTH)
    if tc.get("model_max_length") is not None:
        max_len = min(int(tc["model_max_length"]), max_len)
    normalize = False
    for kind, mdir in module_entries(path):
        if kind == "Dense":
            raise ValueError(f"{path}: Dense module {mdir!r} in a Qwen3 snapshot is not supported: Qwen3 encoders "
                             f"normalise their last-token row themselves and take no projection")
        if kind == "Pooling":
            pc = _read_json(os.path.join(path, mdir, "config.json")) or {}
            other = [k for k, v in pc.items() if k.startswith("pooling_mode_") and v and k != "pooling_mode_lasttoken"]
            if not pc.get("pooling_mode_lasttoken") or other:
                raise ValueError(f"{path}: Qwen3 embedders pool by the last token only; {mdir} asks for "
                                 f"{other or 'no pooling_mode_lasttoken'}")
        if kind == "Normalize":
            normalize = True
    sb = _read_json(os.path.join(path, "sentence_bert_config.json"))
    if sb and sb.get("max_seq_length"):
        max_len = min(int(sb["max_seq_length"]), cfg.max_pos)
    st = _read_json(os.path.join(path, "config_sentence_transformers.json")) or {}
    if st.get("default_prompt_name"):
        cfg.prompt = (st.get("prompts") or {})[st["default_prompt_name"]]
    return cfg, {n: w[n] for n, _ in qwen3_weight_names(cfg, with_head)}, "last", normalize, max_len, act


def _tensor_names_file(st: str):
    from safetensors import safe_open
    with safe_open(st, framework="numpy") as f:
        return set(f.keys())


def resolve_model(model_name: str, with_head: bool, cache_folder: Optional[str] = None):
    """model id -> (cfg, weights, pooling, normalize, max_seq_length, activation, vocab_source).

    ``synthetic:<preset>[:seed[:scale]]`` builds seeded weights; anything else must be a
    local directory (or a directory ``<cache>/<name>`` / ``$RAGMEUP_MODEL_DIR/<name>``)."""
    if model_name.startswith("synthetic:"):
        parts = model_name.split(":")
        preset = parts[1]
        seed = int(parts[2]) if len(parts) > 2 else 0
        scale = float(parts[3]) if len(parts) > 3 else 1.0
        if preset not in PRESETS:
            raise ValueError(f"unknown synthetic preset {preset!r}; have {sorted(PRESETS)}")
        cfg, pooling, max_len = PRESETS[preset]
        if isinstance(cfg, MPNetConfig) and with_head:
            raise ValueError(f"synthetic preset {preset!r} is MPNet: MPNet cross-encoders are not supported")
        if isinstance(cfg, DebertaConfig) and not with_head:
            raise ValueError(f"synthetic preset {preset!r}: model_type 'deberta-v2' runs as a cross-encoder only")
        cfg = type(cfg)(**asdict(cfg))
        if isinstance(cfg, Qwen3Config):
            cfg.name = model_name
            w = synthetic_qwen3_weights(cfg, seed=seed, with_head=with_head, scale=scale)
            act = ("yes_prob" if cfg.reranker else "sigmoid") if with_head else "identity"
            return cfg, w, pooling, preset not in UNNORMALIZED_PRESETS, max_len, act, None
        if isinstance(cfg, XmodConfig):
            cfg.language = select_language(cfg.languages, cfg.language, model_name)
        w = synthetic_bert_weights(cfg, seed=seed, with_head=with_head, scale=scale)
        w.update(synthetic_dense_weights(cfg.hidden, DENSE_PRESETS.get(preset, ()), seed=seed, scale=scale))
        # an XLM-R preset scores as its checkpoint does: one label, no sbert_ce_default_activation_function -> sigmoid
        act = ("sigmoid" if with_head and isinstance(cfg, (XLMRConfig, DebertaConfig, ModernBertConfig, DistilBertConfig))
               and cfg.num_labels == 1 else "identity")
        return cfg, w, pooling, preset not in UNNORMALIZED_PRESETS, max_len, act, None
    c = find_snapshot(model_name, cache_folder)
    return (*load_hf_snapshot(c, with_head), c)


@dataclass
class ColBERTSpec:
    """ColBERT's scoring settings.  The defaults are colbert-ai's ``ColBERTConfig`` defaults [3P-recall: colbert-ai
    0.2.x, not installed here]: query_maxlen 32, doc_maxlen 220, dim 128, markers [unused0] / [unused1],
    attend_to_mask_tokens False, mask_punctuation True, cosine similarity.  A snapshot's ``artifact.metadata`` overrides
    them."""
    dim: int = 128
    query_maxlen: int = 32
    doc_maxlen: int = 220
    query_token: str = "[unused0]"
    doc_token: str = "[unused1]"
    attend_to_mask_tokens: bool = False
    mask_punctuation: bool = True
    similarity: str = "cosine"


# synthetic ColBERT checkpoints: (config, spec).  colbertv2.0 is BERT-base with dim 128, query_maxlen 32 and
# doc_maxlen 180, the values of colbert-ir/colbertv2.0's artifact.metadata [3P-recall].  tiny-colbert has dim = H = 128,
# so a transposed `linear` has the right shape and must be caught by the numbers.
COLBERT_PRESETS: Dict[str, Tuple[BertConfig, ColBERTSpec]] = {
    "colbertv2.0": (BertConfig(hidden=768, layers=12, heads=12, ffn=3072), ColBERTSpec(doc_maxlen=180)),
    "tiny-colbert": (BertConfig(vocab_size=1000, hidden=128, layers=2, heads=4, ffn=256, max_pos=128),
                     ColBERTSpec(query_maxlen=16, doc_maxlen=64)),
    # antoinelouis/colbert-xm, the reference README's multilingual pick: an xmod-base backbone with colbert-ai's default
    # dim and lengths [3P-recall: its artifact.metadata is not read here]; [unused0] / [unused1] are not in XLM-R's
    # vocabulary, so both markers are <unk>
    "colbert-xm": (XmodConfig(hidden=768, layers=12, heads=12, ffn=3072, adapter_dim=384), ColBERTSpec()),
    "tiny-colbert-xm": (XmodConfig(vocab_size=2000, hidden=256, layers=2, heads=4, ffn=512, max_pos=130, adapter_dim=128),
                        ColBERTSpec(query_maxlen=16, doc_maxlen=64)),
}


def colbert_spec(meta: Optional[dict], dim: int) -> ColBERTSpec:
    """``artifact.metadata`` (or None) + the rows of ``linear.weight`` -> ColBERTSpec; refuses what the encoder does
    not compute: a similarity other than cosine, attend_to_mask_tokens, a dim that disagrees with the weight, and a dim
    above 128 that is not a multiple of 128 (the projection runs on 128-column tiles)."""
    meta = meta or {}
    s = ColBERTSpec(dim=int(dim))
    for key, field in (("query_maxlen", "query_maxlen"), ("doc_maxlen", "doc_maxlen"), ("query_token_id", "query_token"),
                       ("doc_token_id", "doc_token"), ("attend_to_mask_tokens", "attend_to_mask_tokens"),
                       ("mask_punctuation", "mask_punctuation"), ("similarity", "similarity")):
        if meta.get(key) is not None:
            setattr(s, field, type(getattr(s, field))(meta[key]))
    if meta.get("dim") is not None and int(meta["dim"]) != s.dim:
        raise ValueError(f"ColBERT: artifact.metadata states dim {meta['dim']} but linear.weight has {s.dim} rows")
    if s.similarity != "cosine":
        raise ValueError(f"ColBERT similarity {s.similarity!r} is not supported (cosine only)")
    if s.attend_to_mask_tokens:
        raise ValueError("ColBERT with attend_to_mask_tokens = true is not supported: the query's [MASK] padding "
                         "attends to the real tokens only")
    if s.dim > 128 and s.dim % 128:
        raise ValueError(f"ColBERT dim {s.dim} is not supported: at most 128, or a multiple of 128")
    return s


def _tensor_names(path: str):
    st = os.path.join(path, "model.safetensors")
    if os.path.exists(st):
        from safetensors import safe_open
        with safe_open(st, framework="numpy") as f:
            return set(f.keys())
    return set(_load_tensors(path))


def is_colbert_snapshot(path: str) -> bool:
    """``architectures`` names HF_ColBERT, or the tensors hold ``linear.weight`` and no classifier"""
    cfgd = _read_json(os.path.join(path, "config.json")) or {}
    if "HF_ColBERT" in (cfgd.get("architectures") or []):
        return True
    names = _tensor_names(path)
    return "linear.weight" in names and not any(n.startswith(("classifier.", "bert.classifier.")) for n in names)


def load_colbert_snapshot(path: str):
    """ColBERT snapshot -> (config, encoder weights without a head, linear [dim, H] fp32, ColBERTSpec).  BERT encoders
    are read under ``bert.`` (or bare); XLM-R, RoBERTa and X-MOD ones under ``roberta.`` (or bare), the base-model prefix
    of transformers' classes for them, which colbert-ai's HF_ColBERT is assumed to keep [3P-recall: colbert-xm's tensor
    names are not read here].  An X-MOD backbone reads only its selected language's adapters.  MPNet is refused."""
    cfgd = _read_json(os.path.join(path, "config.json")) or {}
    kind = cfgd.get("model_type", "bert")
    if kind == "deberta-v2":
        raise ValueError(f"{path}: a ColBERT checkpoint of model_type 'deberta-v2' is not supported: DeBERTa runs as a "
                         f"cross-encoder only")
    if kind == "modernbert":
        raise ValueError(f"{path}: a ColBERT checkpoint of model_type 'modernbert' is not supported: ModernBERT runs as a "
                         f"cross-encoder or an embedder")
    if kind == "qwen3":
        raise ValueError(f"{path}: a ColBERT checkpoint of model_type 'qwen3' is not supported: Qwen3 runs as a "
                         f"cross-encoder or an embedder")
    if kind == "distilbert":
        raise ValueError(f"{path}: a ColBERT checkpoint of model_type 'distilbert' is not supported: DistilBERT runs as a "
                         f"cross-encoder or an embedder")
    if kind not in ("bert", "xlm-roberta", "roberta", "xmod"):
        raise ValueError(f"{path}: a ColBERT checkpoint of model_type {kind!r} is not supported (bert, xlm-roberta, "
                         f"roberta and xmod are)")
    if kind == "bert":
        cfg = BertConfig.from_hf(cfgd)
        raw = _load_tensors(path)
        w = {(k[5:] if k.startswith("bert.") else k): np.ascontiguousarray(v, dtype=np.float32) for k, v in raw.items()}
    else:
        if any(n.startswith("bert.") for n in _tensor_names(path)):
            raise ValueError(f"{path}: a ColBERT checkpoint of model_type {kind!r} holds its encoder under 'bert.'; "
                             f"that prefix is read for BERT only (model_type bert), so the snapshot contradicts itself")
        cfg = XmodConfig.from_hf(cfgd, path) if kind == "xmod" else XLMRConfig.from_hf(cfgd)
        w = xlmr_to_canonical(_load_tensors(path, _xmod_keep(cfg.language) if cfg.adapter_dim else None))
    missing = [n for n, _ in weight_names(cfg, False) if n not in w]
    if missing or "linear.weight" not in w:
        raise KeyError(f"{path}: missing tensors {(missing or ['linear.weight'])[:4]}...")
    lin = w["linear.weight"]
    if lin.ndim != 2 or lin.shape[1] != cfg.hidden:
        raise ValueError(f"{path}: linear.weight has shape {lin.shape}, expected [dim, {cfg.hidden}]")
    spec = colbert_spec(_read_json(os.path.join(path, "artifact.metadata")), lin.shape[0])
    return cfg, {n: w[n] for n, _ in weight_names(cfg, False)}, np.ascontiguousarray(lin), spec


def synthetic_colbert(preset: str, seed: int = 0, scale: float = 1.0):
    """seeded ColBERT weights of a COLBERT_PRESETS shape -> (cfg, weights, linear [dim, H], spec); ``linear`` is
    N(0, 0.02 * scale) like the other projections"""
    cfg, spec = COLBERT_PRESETS[preset]
    cfg = type(cfg)(**asdict(cfg))
    if isinstance(cfg, XmodConfig):
        cfg.language = select_language(cfg.languages, cfg.language, f"synthetic:{preset}")
    w = synthetic_bert_weights(cfg, seed=seed, with_head=False, scale=scale)
    rng = np.random.default_rng(seed + 7919)
    lin = (0.02 * scale * rng.standard_normal((spec.dim, cfg.hidden))).astype(np.float32)
    return cfg, w, lin, ColBERTSpec(**asdict(spec))


def resolve_colbert(model_name: str, cache_folder: Optional[str] = None):
    """model id -> (cfg, weights, linear, spec, vocab_source) when it names a ColBERT checkpoint (``synthetic:`` one of
    COLBERT_PRESETS, or a snapshot found as in ``resolve_model``), else None.  A snapshot whose model_type is not one
    of MODEL_TYPES, and an X-MOD one without a language it can run (``select_language``), is left to
    ``resolve_model``, which refuses it with the same error as any other model of that type."""
    if model_name.startswith("synthetic:"):
        parts = model_name.split(":")
        if parts[1] not in COLBERT_PRESETS:
            return None
        seed = int(parts[2]) if len(parts) > 2 else 0
        scale = float(parts[3]) if len(parts) > 3 else 1.0
        return (*synthetic_colbert(parts[1], seed, scale), None)
    cands = [model_name]
    for root in (cache_folder, os.environ.get("RAGMEUP_MODEL_DIR")):
        if root:
            cands += [os.path.join(root, model_name), os.path.join(root, model_name.split("/")[-1])]
    for c in cands:
        if os.path.isdir(c):
            cfgd = _read_json(os.path.join(c, "config.json"))
            if cfgd is None or cfgd.get("model_type", "bert") not in MODEL_TYPES or cfgd.get("model_type") == "qwen3" \
                    or not is_colbert_snapshot(c):
                return None
            if cfgd.get("model_type") == "xmod":
                try:
                    select_language(xmod_languages(cfgd), cfgd.get("default_language"), c)
                except ValueError:
                    return None
            return (*load_colbert_snapshot(c), c)
    return None


def _refuse_xlmr_flashrank(cfg: BertConfig, where: str) -> None:
    if isinstance(cfg, Qwen3Config):
        raise ValueError(f"{where}: a Qwen3 (model_type 'qwen3') model is not a FlashRank model (FlashRank's rerankers "
                         f"are BERT checkpoints); use HuggingFaceCrossEncoder for it")
    if isinstance(cfg, ModernBertConfig):
        raise ValueError(f"{where}: a ModernBERT (model_type 'modernbert') model is not a FlashRank model (FlashRank's "
                         f"rerankers are BERT checkpoints); use HuggingFaceCrossEncoder for it")
    if isinstance(cfg, DistilBertConfig):
        raise ValueError(f"{where}: a DistilBERT (model_type 'distilbert') model is not a FlashRank model (FlashRank's "
                         f"rerankers are BERT checkpoints); use HuggingFaceCrossEncoder for it")
    if isinstance(cfg, DebertaConfig):
        raise ValueError(f"{where}: a DeBERTa-v2 (model_type 'deberta-v2') model is not a FlashRank model (FlashRank's "
                         f"rerankers are BERT checkpoints); use HuggingFaceCrossEncoder for it")
    if isinstance(cfg, XLMRConfig):
        kind = "an X-MOD" if isinstance(cfg, XmodConfig) else "an XLM-R / RoBERTa"
        raise ValueError(f"{where}: {kind} model is not a FlashRank model (FlashRank's rerankers are BERT "
                         f"checkpoints); use HuggingFaceCrossEncoder for it")


def resolve_flashrank(model_name: str, cache_folder: Optional[str] = None, max_length: int = 512):
    """FlashRank model name -> (cfg, weights with the classifier head, max_length, vocab_source).

    A snapshot is looked up under ``cache_folder`` and ``$RAGMEUP_MODEL_DIR`` by either name: the FlashRank name or
    the HuggingFace id of FLASHRANK_MODELS (``<root>/<org>/<name>`` or ``<root>/<name>``).  ``synthetic:<preset>``
    names work as in ``resolve_model``.  ``num_labels`` is the classifier's row count; a config that states another
    count is refused.  ``max_length`` is FlashRank's truncation [3P-recall]: ``min(model_max_length of
    tokenizer_config.json, max_length)``, or ``min(max_position_embeddings, max_length)`` without that file or key."""
    if model_name.startswith("synthetic:"):
        cfg, w, _pool, _norm, _len, _act, src = resolve_model(model_name, with_head=True)
        _refuse_xlmr_flashrank(cfg, model_name)
        return cfg, w, min(cfg.max_pos, int(max_length)), src
    if model_name not in FLASHRANK_MODELS:
        raise ValueError(f"FlashRank model {model_name!r} is not supported here: the BERT cross-encoders "
                         f"{sorted(FLASHRANK_MODELS)} are (or 'synthetic:<preset>')")
    hf = FLASHRANK_MODELS[model_name]
    names = [model_name, hf, hf.split("/")[-1]]
    roots = [r for r in (cache_folder, os.environ.get("RAGMEUP_MODEL_DIR")) if r]
    path = next((os.path.join(r, n) for r in roots for n in names if os.path.isdir(os.path.join(r, n))), None)
    if path is None:
        raise FileNotFoundError(
            f"FlashRank model {model_name!r} not found locally (no network in this deployment): put the HuggingFace "
            f"snapshot of {hf!r} at <dir>/{model_name} or <dir>/{hf}, with <dir> = RAGMEUP_MODEL_DIR or cache_folder "
            f"(searched: {roots or 'none set'})")
    cfgd = _read_json(os.path.join(path, "config.json")) or {}
    cfg, w, *_ = load_hf_snapshot(path, with_head=True)
    _refuse_xlmr_flashrank(cfg, path)
    rows = int(w["classifier.weight"].shape[0])
    stated = len(cfgd["id2label"]) if "id2label" in cfgd else cfgd.get("num_labels")
    if stated is not None and int(stated) != rows:
        raise ValueError(f"{path}: the classifier has {rows} rows but config.json states {stated} labels")
    cfg.num_labels = rows
    tc = _read_json(os.path.join(path, "tokenizer_config.json")) or {}
    if tc.get("model_max_length") is not None:
        max_len = min(int(tc["model_max_length"]), int(max_length))
    else:
        max_len = min(cfg.max_pos, int(max_length))
    return cfg, w, min(max_len, cfg.max_pos), path     # the model has no positions past max_pos
