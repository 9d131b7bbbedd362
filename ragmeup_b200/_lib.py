"""ctypes binding of libragmeup_b200.so — the ONLY way the Python host code reaches the GPU.

There is no CPU fallback: if the library is missing or no CUDA device is present every product
call raises.  (``include/ragmeup_b200.h`` is the authoritative declaration of these symbols.)
"""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libragmeup_b200.so")

_lock = threading.Lock()
_lib = None


class RmuError(RuntimeError):
    pass


class BertConfigC(C.Structure):
    _fields_ = [("vocab_size", C.c_int32), ("hidden", C.c_int32), ("layers", C.c_int32), ("heads", C.c_int32),
                ("ffn", C.c_int32), ("max_pos", C.c_int32), ("type_vocab", C.c_int32), ("num_labels", C.c_int32),
                ("ln_eps", C.c_float), ("position_mode", C.c_int32), ("rel_buckets", C.c_int32),
                ("adapter_dim", C.c_int32)]


class EncoderExtC(C.Structure):
    _fields_ = [("position_buckets", C.c_int32), ("max_relative_positions", C.c_int32), ("head_act", C.c_int32)]


class ModernBertExtC(C.Structure):
    _fields_ = [("half_window_h", C.c_void_p), ("pooling", C.c_int32), ("head_form", C.c_int32), ("rope_rows", C.c_int32),
                ("rope_half", C.c_int32)]


class Qwen3ExtC(C.Structure):
    _fields_ = [("kv_heads", C.c_int32), ("head_dim", C.c_int32), ("rope_rows", C.c_int32), ("rope_half", C.c_int32),
                ("head_form", C.c_int32), ("pad_token_id", C.c_int32)]


MAX_EOS = 8
MAX_GENERATE_BATCH = 16            # RMU_MAX_GENERATE_BATCH
ERR_RANGE = -4                     # RMU_ERR_RANGE
ERR_BUSY = -5                      # RMU_ERR_BUSY
GEN_LIVE, GEN_EOS, GEN_MAX_NEW, GEN_MAX_POS = 0, 1, 2, 3   # RMU_GEN_*: a session row's status


class SamplingC(C.Structure):
    _fields_ = [("do_sample", C.c_int32), ("temperature", C.c_float), ("top_p", C.c_float),
                ("repetition_penalty", C.c_float), ("top_k", C.c_int32), ("n_eos", C.c_int32),
                ("eos_ids", C.c_int32 * MAX_EOS)]


def bert_config_c(cfg) -> BertConfigC:
    """weights.BertConfig (or a subclass) -> the C struct; adapter_dim is 0 for every family but X-MOD"""
    return BertConfigC(cfg.vocab_size, cfg.hidden, cfg.layers, cfg.heads, cfg.ffn, cfg.max_pos, cfg.type_vocab,
                       cfg.num_labels, cfg.ln_eps, cfg.position_mode, cfg.rel_buckets, cfg.adapter_dim)


def encoder_ext_c(cfg) -> EncoderExtC:
    """rmu_encoder_create_ex's extra fields: DeBERTa-v2's buckets and head activation, zero for every other family"""
    return EncoderExtC(cfg.position_buckets, cfg.max_relative_positions, cfg.head_act)


# name -> (restype, argtypes); mirrors include/ragmeup_b200.h
SIGNATURES = {
    "rmu_last_error": (C.c_char_p, []),
    "rmu_version": (C.c_int, []),
    "rmu_launch_count": (C.c_uint64, []),
    "rmu_profile_enable": (None, [C.c_int]),
    "rmu_profile_reset": (None, []),
    "rmu_profile_read": (C.c_int, [C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
    "rmu_index_create": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "rmu_index_destroy": (None, [C.c_void_p]),
    "rmu_index_reserve": (C.c_int, [C.c_void_p, C.c_int64]),
    "rmu_index_add": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]),
    "rmu_index_set_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "rmu_index_remove": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "rmu_index_size": (C.c_int64, [C.c_void_p]),
    "rmu_index_dim": (C.c_int, [C.c_void_p]),
    "rmu_index_metric": (C.c_int, [C.c_void_p]),
    "rmu_index_clear": (C.c_int, [C.c_void_p]),
    "rmu_index_data": (C.c_void_p, [C.c_void_p]),
    "rmu_index_search": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_index_search_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_void_p]),
    "rmu_debug_scan_tile": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "rmu_index_gather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "rmu_topk_merge": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                 C.c_void_p]),
    "rmu_topk_merge_strided": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_adjacent_cosine_distance": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "rmu_mmr_select": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double,
                                 C.c_void_p, C.c_void_p]),
    "rmu_bm25_create": (C.c_int, [C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_double, C.POINTER(C.c_void_p)]),
    "rmu_bm25_destroy": (C.c_int, [C.c_void_p]),
    "rmu_bm25_size": (C.c_int64, [C.c_void_p]),
    "rmu_bm25_terms": (C.c_int64, [C.c_void_p]),
    "rmu_bm25_search": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                  C.c_void_p]),
    "rmu_bm25_search_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_void_p]),
    "rmu_bm25_csr_build": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_void_p)]),
    "rmu_bm25_csr_sizes": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "rmu_bm25_csr_export": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p]),
    "rmu_bm25_csr_free": (C.c_int, [C.c_void_p]),
    "rmu_pgbm25_create": (C.c_int, [C.POINTER(C.c_void_p)]),
    "rmu_pgbm25_destroy": (C.c_int, [C.c_void_p]),
    "rmu_pgbm25_push_segment": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_pgbm25_pop_segments": (C.c_int, [C.c_void_p, C.c_int]),
    "rmu_pgbm25_segments": (C.c_int, [C.c_void_p]),
    "rmu_pgbm25_set_alive": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64]),
    "rmu_pgbm25_search_host": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_encoder_create": (C.c_int, [C.POINTER(BertConfigC), C.POINTER(C.c_void_p), C.c_int, C.c_int,
                                     C.POINTER(C.c_void_p)]),
    "rmu_encoder_create_ex": (C.c_int, [C.POINTER(BertConfigC), C.POINTER(EncoderExtC), C.POINTER(C.c_void_p), C.c_int,
                                        C.c_int, C.POINTER(C.c_void_p)]),
    "rmu_encoder_create_modernbert": (C.c_int, [C.POINTER(BertConfigC), C.POINTER(ModernBertExtC), C.POINTER(C.c_void_p),
                                                C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "rmu_encoder_create_qwen3": (C.c_int, [C.POINTER(BertConfigC), C.POINTER(Qwen3ExtC), C.POINTER(C.c_void_p), C.c_int,
                                           C.c_int, C.POINTER(C.c_void_p)]),
    "rmu_encoder_create_llama": (C.c_int, [C.POINTER(BertConfigC), C.POINTER(Qwen3ExtC), C.POINTER(C.c_void_p), C.c_int,
                                           C.POINTER(C.c_void_p)]),
    "rmu_decoder_attention_spans": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                              C.c_void_p]),
    "rmu_decoder_set_lm_head": (C.c_int, [C.c_void_p, C.c_void_p]),
    "rmu_decoder_quantize_nf4": (C.c_int, [C.c_void_p, C.c_void_p]),
    "rmu_decoder_create_nf4": (C.c_int, [C.POINTER(BertConfigC), C.POINTER(Qwen3ExtC), C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "rmu_decoder_load_layer_nf4": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.c_void_p]),
    "rmu_decoder_generate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(SamplingC), C.c_uint64, C.c_int,
                                       C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.c_void_p]),
    "rmu_decoder_generate_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(SamplingC),
                                             C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_decoder_generate_lookup": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(SamplingC), C.c_uint64, C.c_int,
                                              C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p,
                                              C.POINTER(C.c_int32), C.c_void_p]),
    "rmu_prompt_lookup_draft": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "rmu_decoder_generate_assisted": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(SamplingC),
                                                C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int32),
                                                C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                                C.POINTER(C.c_int32), C.c_void_p]),
    "rmu_decoder_session_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "rmu_decoder_session_destroy": (None, [C.c_void_p]),
    "rmu_decoder_session_add": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_decoder_session_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32),
                                           C.c_void_p, C.c_void_p]),
    "rmu_decoder_session_cancel": (C.c_int, [C.c_void_p, C.c_int]),
    "rmu_decoder_session_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                           C.POINTER(C.c_uint32)]),
    "rmu_debug_kv_regions": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "rmu_encoder_destroy": (None, [C.c_void_p]),
    "rmu_encoder_embed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_int, C.c_void_p, C.c_void_p]),
    "rmu_encoder_classify": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                       C.c_void_p, C.c_void_p]),
    "rmu_encoder_hidden": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                     C.c_void_p, C.c_void_p]),
    "rmu_encoder_embed_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                         C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "rmu_encoder_classify_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                            C.c_void_p, C.c_void_p]),
    "rmu_encoder_set_dense": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                        C.c_void_p]),
    "rmu_colbert_create": (C.c_int, [C.POINTER(BertConfigC), C.POINTER(C.c_void_p), C.c_int, C.c_void_p, C.c_int,
                                     C.POINTER(C.c_void_p)]),
    "rmu_colbert_destroy": (None, [C.c_void_p]),
    "rmu_colbert_dim": (C.c_int, [C.c_void_p]),
    "rmu_colbert_vectors": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                      C.c_int, C.c_void_p, C.c_void_p]),
    "rmu_colbert_maxsim": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                     C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "rmu_colbert_score_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_int, C.c_void_p, C.c_void_p]),
    "rmu_debug_attention_keys": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                           C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_gemm": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                 C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_layernorm": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p,
                                      C.c_void_p, C.c_void_p]),
    "rmu_debug_embed_ln": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float,
                                     C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_embed_ln_pos": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float,
                                         C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_relative_bias_table": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "rmu_debug_attention_bias": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                           C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_log_bucket_table": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "rmu_debug_attention_disentangled": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                   C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                                   C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_encoder_position_planes": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_cls_head_act": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "rmu_debug_dense": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                  C.c_void_p, C.c_void_p]),
    "rmu_debug_pool": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                 C.c_void_p]),
    "rmu_debug_cls_head": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_gemm_ex": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                    C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p]),
    "rmu_debug_attention_window": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_modernbert_head": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_gemm_swiglu": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                        C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_rmsnorm": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p]),
    "rmu_debug_qk_norm_rope": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p]),
    "rmu_debug_attention_causal": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_attention_spans": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                            C.c_void_p, C.c_void_p]),
    "rmu_debug_last_token": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_float,
                                       C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "rmu_debug_attention_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_attention_decode_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int,
                                                  C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                  C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_attention_cached": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                             C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_sample_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                        C.POINTER(SamplingC), C.c_void_p, C.c_void_p]),
    "rmu_debug_sample_verify_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64,
                                               C.c_int64, C.POINTER(SamplingC), C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_sample_session_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_generate_drafts": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(SamplingC), C.c_uint64, C.c_int,
                                            C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p,
                                            C.POINTER(C.c_int32), C.c_void_p]),
    "rmu_debug_kv_append": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                      C.c_void_p]),
    "rmu_debug_nf4_quantize": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_nf4_dequantize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "rmu_debug_nf4_gemv": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_nf4_gemv_rows": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                          C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p]),
    "rmu_debug_nf4_conversion": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "rmu_debug_sample": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.POINTER(SamplingC), C.c_float, C.c_void_p,
                                   C.c_void_p]),
    "rmu_debug_split_planes": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rmu_debug_join_planes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "rmu_debug_bm25_select": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
}


def lib() -> C.CDLL:
    """Load (once) and return the shared library with typed signatures."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            # the library is built in-tree and normally travels with the checkout; build it when absent
            try:
                from . import build as _build
                _build.build()
            except Exception as e:  # noqa: BLE001
                raise RmuError(f"{LIB_PATH} is not built and building it failed ({e}): run "
                               f"`python -m ragmeup_b200.build` (there is no CPU fallback for this path)") from e
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().rmu_last_error()
        raise RmuError(f"{what or 'ragmeup_b200'} failed (rc={rc}): {msg.decode() if msg else '?'}")


def launch_count() -> int:
    return int(lib().rmu_launch_count())


def require_cuda():
    """The product path is CUDA-only (the reference's force_cpu / device='cpu' has no equivalent)."""
    import torch
    if not torch.cuda.is_available():
        raise RmuError("ragmeup_b200 needs a CUDA device (sm_90a); there is no CPU path")
    return torch


def stream_ptr(torch_stream=None) -> int:
    import torch
    s = torch_stream if torch_stream is not None else torch.cuda.current_stream()
    return int(s.cuda_stream)


PROF_CLASSES = ["scan", "finalize", "exact", "merge", "gemm", "attention", "layernorm", "embedding", "pool_head", "misc",
                "scan_pass2"]


def profile_enable(on: bool) -> None:
    lib().rmu_profile_enable(int(bool(on)))


def profile_reset() -> None:
    lib().rmu_profile_reset()


def profile_read() -> dict:
    """{class: (total_ms, launches)} since the last reset (synchronises the recorded events)."""
    out = {}
    for i, name in enumerate(PROF_CLASSES):
        ms, n = C.c_double(0), C.c_int64(0)
        check(lib().rmu_profile_read(i, C.byref(ms), C.byref(n)), "rmu_profile_read")
        out[name] = (ms.value, int(n.value))
    return out
