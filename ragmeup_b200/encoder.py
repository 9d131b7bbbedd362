"""BertEncoder — torch/numpy view of the C-ABI BERT encoder (``rmu_encoder_*``).

Weights go to the library in the canonical order of ``weights.weight_names`` (HuggingFace
``BertModel`` tensor order: embeddings, then per layer q/k/v/attention-output/LayerNorm/
intermediate/output/LayerNorm, then pooler + classifier when a head is present, then MPNet's
relative attention bias [32, heads] when the config has one, then X-MOD's language adapter of every layer, for the
config's one language, when it has ``adapter_dim > 0``, then DeBERTa's relative embeddings and LN_rel when it has
``position_buckets > 0``).

ModernBERT takes its own order (``weights.modernbert_weight_names``, ``rmu_encoder_create_modernbert``): the token
embeddings and their norm; per layer attn_norm (layer 0: placeholders, not read), Wqkv, Wo, mlp_norm, Wi, mlp Wo, each
with its bias (zeros where the checkpoint has none); final_norm; with a head, head.dense, head.norm and the classifier;
then the four rope tables of ``weights.rope_tables``, computed here from the config.

Qwen3 takes its own order too (``weights.qwen3_weight_names``, ``rmu_encoder_create_qwen3``): embed_tokens; per layer
input_layernorm, q / k / v_proj, q_norm, k_norm, o_proj, post_attention_layernorm, gate / up / down_proj; norm; with a
head the [num_labels, H] last-token head; then the cos / sin tables of ``weights.rope_table``.  It pools by the last
token only (``pooling="last"``), and a forward whose activations leave the fp16 range of the split planes raises
``RmuError`` naming the model.

Llama (``weights.LlamaConfig``, ``rmu_encoder_create_llama``) takes Qwen3's order without q_norm / k_norm and without a
head, with the config's own rope tables (``llama3`` scaling); it is built for attention provenance only.

A weight dict that holds sentence-transformers Dense modules (``weights.dense_layers``) attaches them to the handle
(``rmu_encoder_set_dense``): the embed entry points then return ``embed_dim`` = the last Dense width per row.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np

from . import _lib
from .weights import (BertConfig, LlamaConfig, ModernBertConfig, Qwen3Config, dense_layers, rope_table, rope_tables,
                      weight_names)

POOL = {"mean": 0, "cls": 1, "last": 2}
RMU_ERR_RANGE = -4
MAX_TOKENS_PER_CALL = 131072    # bounds the activation workspace (~19 KB/token for MiniLM shapes => ~2.5 GB)
POSITION_WS_BYTES = 1 << 30     # DeBERTa: bound of the attention position terms' workspace, 2 T heads W fp32 per call


def deberta_tokens_per_call(cfg: BertConfig) -> int:
    """tokens per encoder call that keep DeBERTa's position terms (C2P and P2C, heads x W floats per token each, W at
    most 2s relative positions) within POSITION_WS_BYTES; MAX_TOKENS_PER_CALL for every other model"""
    if not cfg.position_buckets:
        return MAX_TOKENS_PER_CALL
    per_token = 2 * cfg.heads * 2 * cfg.position_buckets * 4
    return max(1, min(MAX_TOKENS_PER_CALL, POSITION_WS_BYTES // per_token))


class BertEncoder:
    def __init__(self, cfg: BertConfig, weights: Dict[str, np.ndarray], with_head: bool, device: Optional[int] = None):
        torch = _lib.require_cuda()
        self.torch = torch
        self.cfg = cfg
        self.with_head = bool(with_head)
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.max_tokens_per_call = deberta_tokens_per_call(cfg)
        names = weight_names(cfg, with_head)
        arrs = []
        for name, shape in names:
            a = np.ascontiguousarray(weights[name], dtype=np.float32)
            if tuple(a.shape) != tuple(shape):
                raise ValueError(f"{name}: expected shape {shape}, got {a.shape}")
            arrs.append(a)
        modern, qwen, llama = isinstance(cfg, ModernBertConfig), isinstance(cfg, Qwen3Config), isinstance(cfg, LlamaConfig)
        if modern:
            arrs += list(rope_tables(cfg))
        if qwen:
            arrs += list(rope_table(cfg.rope_theta, cfg.head_dim, cfg.max_pos))
        if llama:
            if self.with_head:
                raise ValueError(f"{cfg.name}: Llama runs without a head")
            arrs += list(cfg.rope_tables())
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        cc = _lib.bert_config_c(cfg)
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            if llama:
                qx = _lib.Qwen3ExtC(cfg.kv_heads, cfg.head_dim, cfg.max_pos, cfg.head_dim // 2, 0, -1)
                _lib.check(_lib.lib().rmu_encoder_create_llama(C.byref(cc), C.byref(qx), ptrs, len(arrs), C.byref(self._h)),
                           "rmu_encoder_create_llama")
            elif qwen:
                qx = _lib.Qwen3ExtC(cfg.kv_heads, cfg.head_dim, cfg.max_pos, cfg.head_dim // 2, int(self.with_head),
                                    cfg.head_pad_id)
                _lib.check(_lib.lib().rmu_encoder_create_qwen3(C.byref(cc), C.byref(qx), ptrs, len(arrs), int(self.with_head),
                                                               C.byref(self._h)), "rmu_encoder_create_qwen3")
            elif modern:
                win = np.ascontiguousarray(cfg.layer_windows, dtype=np.int32)
                mb = _lib.ModernBertExtC(win.ctypes.data, POOL[cfg.classifier_pooling], 0, cfg.max_pos, cfg.head_dim // 2)
                _lib.check(_lib.lib().rmu_encoder_create_modernbert(C.byref(cc), C.byref(mb), ptrs, len(arrs),
                                                                    int(self.with_head), C.byref(self._h)),
                           "rmu_encoder_create_modernbert")
            else:
                ext = _lib.encoder_ext_c(cfg)
                _lib.check(_lib.lib().rmu_encoder_create_ex(C.byref(cc), C.byref(ext), ptrs, len(arrs), int(self.with_head),
                                                            C.byref(self._h)), "rmu_encoder_create_ex")
            dense = dense_layers(weights)
            self.embed_dim = int(dense[-1][0].shape[0]) if dense else cfg.hidden
            if dense:
                Ws = [np.ascontiguousarray(W, dtype=np.float32) for W, _b, _a in dense]
                bs = [None if b is None else np.ascontiguousarray(b, dtype=np.float32) for _W, b, _a in dense]
                dims = np.asarray([cfg.hidden] + [W.shape[0] for W in Ws], dtype=np.int32)
                acts = np.asarray([a for _W, _b, a in dense], dtype=np.int32)
                _lib.check(_lib.lib().rmu_encoder_set_dense(
                    self._h, len(Ws), dims.ctypes.data, (C.c_void_p * len(Ws))(*[W.ctypes.data for W in Ws]),
                    (C.c_void_p * len(bs))(*[None if b is None else b.ctypes.data for b in bs]), acts.ctypes.data),
                    "rmu_encoder_set_dense")

    @classmethod
    def nf4_decoder(cls, layers, device: Optional[int] = None, on_layer=None) -> "BertEncoder":
        """a Llama or Qwen3 decoder in NF4 built one layer at a time from ``layers`` (``weights.DecoderLayers``):
        ``rmu_decoder_create_nf4`` with the embeddings, final norm and rope tables, then ``rmu_decoder_load_layer_nf4``
        per layer, so host memory holds the embeddings and one layer, and the device the finished handle and one
        staging chunk.  ``on_layer(l)``, when given, runs after layer l is loaded."""
        torch = _lib.require_cuda()
        cfg = layers.cfg
        llama = isinstance(cfg, LlamaConfig)
        if not llama and not isinstance(cfg, Qwen3Config):
            raise ValueError(f"{getattr(cfg, 'name', 'model')}: NF4 decoders are Llama or Qwen3")
        self = cls.__new__(cls)
        self.torch = torch
        self.cfg = cfg
        self.with_head = False
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.max_tokens_per_call = MAX_TOKENS_PER_CALL
        self.embed_dim = cfg.hidden
        self._h = C.c_void_p()

        def f32(a, shape, name):
            a = np.ascontiguousarray(a, dtype=np.float32)
            if tuple(a.shape) != tuple(shape):
                raise ValueError(f"{name}: expected shape {shape}, got {a.shape}")
            return a
        g = layers.globals()
        embed = f32(g["embed_tokens.weight"], (cfg.vocab_size, cfg.hidden), "embed_tokens.weight")
        norm = f32(g["norm.weight"], (cfg.hidden,), "norm.weight")
        cos, sin = cfg.rope_tables() if llama else rope_table(cfg.rope_theta, cfg.head_dim, cfg.max_pos)
        cos, sin = np.ascontiguousarray(cos, dtype=np.float32), np.ascontiguousarray(sin, dtype=np.float32)
        cc = _lib.bert_config_c(cfg)
        qx = _lib.Qwen3ExtC(cfg.kv_heads, cfg.head_dim, cfg.max_pos, cfg.head_dim // 2, 0, -1)
        lib = _lib.lib()
        with torch.cuda.device(self.device):
            _lib.check(lib.rmu_decoder_create_nf4(C.byref(cc), C.byref(qx), int(not llama), embed.ctypes.data,
                                                  norm.ctypes.data, cos.ctypes.data, sin.ctypes.data, C.byref(self._h)),
                       "rmu_decoder_create_nf4")
            del embed, g
            for l in range(cfg.layers):
                t = layers.layer(l)
                arrs = [f32(t[n], shape, n) for n, shape in layers.layer_names(l)]
                del t
                ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
                _lib.check(lib.rmu_decoder_load_layer_nf4(self._h, l, ptrs, _lib.stream_ptr()),
                           "rmu_decoder_load_layer_nf4")
                del arrs
                if on_layer is not None:
                    on_layer(l)
        return self

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                _lib.lib().rmu_encoder_destroy(h)
            except Exception:
                pass
            self._h = C.c_void_p()

    def _check(self, rc: int, what: str) -> None:
        """``_lib.check``; an activation that left the fp16 range (Qwen3) raises naming the model"""
        if rc == RMU_ERR_RANGE:
            msg = _lib.lib().rmu_last_error()
            raise _lib.RmuError(f"{getattr(self.cfg, 'name', 'model')}: {what} failed: {msg.decode() if msg else '?'}")
        _lib.check(rc, what)

    # ------------------------------------------------------------------ device-tensor entry points
    def _dev(self, a, dtype):
        torch = self.torch
        if isinstance(a, np.ndarray):
            a = torch.from_numpy(np.ascontiguousarray(a))
        return a.to(device=self.device, dtype=dtype, non_blocking=True).contiguous()

    def _run_tokens(self, name: str, ids, type_ids, cu_seqlens, max_seqlen: int, width: int, *args, per_token=False):
        """the ragged batch as CUDA int32 tensors -> the rmu_encoder_<name> entry point -> CUDA fp32 [B, width], or
        [total_tokens, width] with per_token; ``args`` go between max_seqlen and the output"""
        torch = self.torch
        ids = self._dev(ids, torch.int32)
        typ = None if type_ids is None else self._dev(type_ids, torch.int32)
        cu = self._dev(cu_seqlens, torch.int32)
        B, T = cu.numel() - 1, ids.numel()
        out = torch.empty((T if per_token else B, width), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            self._check(getattr(_lib.lib(), name)(self._h, ids.data_ptr(), None if typ is None else typ.data_ptr(),
                                                  cu.data_ptr(), B, T, int(max_seqlen), *args, out.data_ptr(),
                                                  _lib.stream_ptr()), name)
        return out

    def embed_tokens(self, ids, type_ids, cu_seqlens, max_seqlen: int, pooling: str = "mean", normalize: bool = True):
        """ragged token batch -> CUDA fp32 [B, embed_dim] sentence embeddings."""
        return self._run_tokens("rmu_encoder_embed", ids, type_ids, cu_seqlens, max_seqlen, self.embed_dim, POOL[pooling],
                                int(bool(normalize)))

    def classify_tokens(self, ids, type_ids, cu_seqlens, max_seqlen: int):
        """ragged (pair) token batch -> CUDA fp32 [B, num_labels] raw logits."""
        return self._run_tokens("rmu_encoder_classify", ids, type_ids, cu_seqlens, max_seqlen, self.cfg.num_labels)

    def hidden_tokens(self, ids, type_ids, cu_seqlens, max_seqlen: int):
        """last hidden state, CUDA fp32 [total_tokens, hidden]."""
        return self._run_tokens("rmu_encoder_hidden", ids, type_ids, cu_seqlens, max_seqlen, self.cfg.hidden, per_token=True)

    # ------------------------------------------------------------------ host-buffer entry points
    @staticmethod
    def _chunks(cu: np.ndarray, max_tokens: int):
        """split sequences [0, B) into runs whose token count stays under max_tokens"""
        B = len(cu) - 1
        s = 0
        while s < B:
            e = s + 1
            while e < B and cu[e + 1] - cu[s] <= max_tokens:
                e += 1
            yield s, e
            s = e

    def _run_host(self, name: str, ids: np.ndarray, type_ids: Optional[np.ndarray], cu: np.ndarray, width: int,
                  *args) -> np.ndarray:
        """host int32 token batch -> the rmu_encoder_<name> entry point (H2D/D2H inside the C call), in runs of at most
        max_tokens_per_call tokens -> host fp32 [B, width]; ``args`` go between max_seqlen and the output"""
        B = len(cu) - 1
        out = np.empty((B, width), dtype=np.float32)
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        typ = None if type_ids is None else np.ascontiguousarray(type_ids, dtype=np.int32)
        cu = np.ascontiguousarray(cu, dtype=np.int32)
        fn = getattr(_lib.lib(), name)
        with self.torch.cuda.device(self.device):
            for s, e in self._chunks(cu, self.max_tokens_per_call):
                t0, t1 = int(cu[s]), int(cu[e])
                sub_cu = np.ascontiguousarray(cu[s:e + 1] - cu[s], dtype=np.int32)
                sub_ids = ids[t0:t1]
                sub_typ = None if typ is None else typ[t0:t1]
                o = out[s:e]
                maxlen = int(np.max(np.diff(sub_cu)))
                self._check(fn(self._h, sub_ids.ctypes.data, None if sub_typ is None else sub_typ.ctypes.data,
                               sub_cu.ctypes.data, e - s, t1 - t0, maxlen, *args, o.ctypes.data, _lib.stream_ptr()), name)
        return out

    def embed_host(self, ids: np.ndarray, type_ids: Optional[np.ndarray], cu: np.ndarray, pooling: str = "mean",
                   normalize: bool = True) -> np.ndarray:
        """host int32 token batch -> host fp32 [B, embed_dim] (H2D/D2H inside the C call)."""
        return self._run_host("rmu_encoder_embed_host", ids, type_ids, cu, self.embed_dim, POOL[pooling],
                              int(bool(normalize)))

    def classify_host(self, ids: np.ndarray, type_ids: Optional[np.ndarray], cu: np.ndarray) -> np.ndarray:
        """host int32 pair-token batch -> host fp32 [B, num_labels] raw logits."""
        return self._run_host("rmu_encoder_classify_host", ids, type_ids, cu, self.cfg.num_labels)
