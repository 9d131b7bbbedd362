"""CPU: the C-ABI library builds, loads, and exports every symbol include/ragmeup_b200.h declares
(no compute calls here — there is no GPU in the build container)."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    from ragmeup_b200 import build
    path = build.build()
    assert os.path.exists(path)
    return path


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "ragmeup_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(rmu_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_path():
    syms = declared_symbols()
    for must in ("rmu_index_create", "rmu_index_add", "rmu_index_search", "rmu_index_search_host", "rmu_topk_merge",
                 "rmu_mmr_select", "rmu_index_gather", "rmu_encoder_create", "rmu_encoder_embed",
                 "rmu_encoder_classify", "rmu_encoder_embed_host", "rmu_encoder_classify_host", "rmu_last_error",
                 "rmu_debug_bm25_select"):
        assert must in syms


def test_library_exports_every_declared_symbol(built_lib):
    lib = ctypes.CDLL(built_lib)
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, missing


def test_loader_signatures_cover_header(built_lib):
    from ragmeup_b200 import _lib
    assert sorted(_lib.SIGNATURES) == declared_symbols()
    l = _lib.lib()
    assert l.rmu_version() >= 100
    assert isinstance(_lib.launch_count(), int)


def test_kernel_test_entry_points_reject_before_any_cuda_call(built_lib):
    """rmu_debug_*: shapes the kernels do not take are refused before a tensor map is encoded or a kernel launched,
    so these run without a device; the pointers are never dereferenced"""
    from ragmeup_b200 import _lib
    l = _lib.lib()
    p = 1 << 20                                    # stand-in device address, never touched

    def gemm(mode=0, a_rows=256, M=200, N=256, K=128, **kw):
        a = dict(res=p, out_f32=p, out_hi=p, out_lo=p, max_ctas=0)
        a.update(kw)
        return l.rmu_debug_gemm(mode, p, p, a_rows, p, p, M, N, K, p, a["res"], a["res"], 0, 1.0, a["max_ctas"],
                                a["out_f32"], a["out_hi"], a["out_lo"], None)

    for mode in range(4):
        assert gemm(mode, N=192) == -3                      # N % 128
        assert gemm(mode, N=64) == -3
        assert gemm(mode, K=96) == -3                       # K % 64
        assert gemm(mode, K=32) == -3
        assert gemm(mode, a_rows=199) == -3                 # A's tensor map must cover M rows
    assert gemm(4) == -1 and gemm(-1) == -1                 # mode
    assert gemm(0, M=0) == -1 and gemm(0, K=0) == -1 and gemm(0, max_ctas=-1) == -1
    assert gemm(0, out_f32=None) == -1 and gemm(2, res=None) == -1
    assert gemm(1, out_hi=None) == -1 and gemm(3, out_lo=None) == -1
    assert gemm(0, N=100) == -3 and b"shape not supported" in l.rmu_last_error()

    def attn(B=2, H=384, heads=12, max_seqlen=64, warps=10, cu=p):
        return l.rmu_debug_attention(p, p, cu, B, H, heads, max_seqlen, warps, p, p, None)

    assert attn(H=384, heads=8) == -3                       # d_h = 48
    assert attn(H=384, heads=4) == -3                       # d_h = 96
    assert attn(H=100, heads=3) == -3
    assert attn(H=768, heads=12, warps=5) == -1             # warps must be 10
    assert attn(H=384, heads=12, warps=5) == -1
    assert attn(warps=7) == -1 and attn(warps=0) == -1
    assert attn(B=0) == -1 and attn(max_seqlen=0) == -1 and attn(cu=None) == -1

    def ln(T=9, H=384):
        return l.rmu_debug_layernorm(p, T, H, p, p, 1e-12, p, p, None)

    assert ln(H=320) == -3 and ln(H=1152) == -3 and ln(H=96) == -3
    assert ln(T=0) == -1

    def emb(B=2, T=9, H=384, vocab=30522, max_pos=512, type_vocab=2, **kw):
        a = dict(ids=p, typ=p, cu=p, word=p, pos=p, ttab=p, g=p, b=p, oh=p, ol=p)
        a.update(kw)
        return l.rmu_debug_embed_ln(a["ids"], a["typ"], a["cu"], B, T, H, vocab, max_pos, type_vocab, a["word"], a["pos"],
                                    a["ttab"], a["g"], a["b"], 1e-12, a["oh"], a["ol"], None)

    assert emb(H=320) == -3 and emb(H=1152) == -3 and emb(H=96) == -3 and b"rmu_debug_embed_ln" in l.rmu_last_error()
    for name in ("ids", "cu", "word", "pos", "ttab", "g", "b", "oh", "ol"):
        assert emb(**{name: None}) == -1, name
    for name in ("B", "T", "vocab", "max_pos", "type_vocab"):
        assert emb(**{name: 0}) == -1 and emb(**{name: -1}) == -1, name
    assert emb(H=0) == -1

    def pool(B=2, H=384, mode=0, hi=p, lo=p, cu=p, out=p):
        return l.rmu_debug_pool(hi, lo, cu, B, H, mode, 1, out, None)

    assert pool(H=1025) == -3 and pool(H=2048) == -3 and b"rmu_debug_pool" in l.rmu_last_error()
    assert pool(mode=2) == -1 and pool(mode=-1) == -1 and pool(B=0) == -1 and pool(H=0) == -1
    assert pool(hi=None) == -1 and pool(lo=None) == -1 and pool(cu=None) == -1 and pool(out=None) == -1

    def head(B=2, H=384, L=1, **kw):
        a = dict(hi=p, lo=p, cu=p, pw=p, pb=p, cw=p, cb=p, out=p)
        a.update(kw)
        return l.rmu_debug_cls_head(a["hi"], a["lo"], a["cu"], B, H, L, a["pw"], a["pb"], a["cw"], a["cb"], a["out"], None)

    assert head(H=1025) == -3 and b"rmu_debug_cls_head" in l.rmu_last_error()
    assert head(B=0) == -1 and head(H=0) == -1 and head(L=0) == -1 and head(L=-2) == -1
    for name in ("hi", "lo", "cu", "pw", "pb", "cw", "cb", "out"):
        assert head(**{name: None}) == -1, name

    assert l.rmu_debug_split_planes(p, -1, p, p, None) == -1 and l.rmu_debug_join_planes(p, p, -1, p, None) == -1
    assert l.rmu_debug_split_planes(None, 8, p, p, None) == -1 and l.rmu_debug_split_planes(p, 8, None, p, None) == -1
    assert l.rmu_debug_split_planes(p, 8, p, None, None) == -1 and l.rmu_debug_join_planes(None, p, 8, p, None) == -1
    assert l.rmu_debug_join_planes(p, None, 8, p, None) == -1 and l.rmu_debug_join_planes(p, p, 8, None, None) == -1
    n0 = _lib.launch_count()                                # n = 0: nothing to launch, so no device is needed
    assert l.rmu_debug_split_planes(p, 0, p, p, None) == 0 and l.rmu_debug_join_planes(p, p, 0, p, None) == 0
    assert _lib.launch_count() == n0

    # the scan tile needs an index handle, which needs a device: what is checked here is refused before the handle is
    # read (the dim / nq / empty-index refusals are in tests/test_index_kernels_gpu.py)
    def tile(h=None, q=p, nq=16, out=p):
        return l.rmu_debug_scan_tile(h, q, nq, out, None)

    assert tile() == -1 and b"rmu_debug_scan_tile" in l.rmu_last_error()
    fake = ctypes.c_void_p(p)                               # never dereferenced: every call below is refused first
    assert tile(fake, q=None) == -1 and tile(fake, out=None) == -1
    assert tile(fake, nq=0) == -1 and tile(fake, nq=-3) == -1 and tile(fake, nq=65) == -1
    assert tile(fake, q=p + 4) == -1 and tile(fake, q=p + 8) == -1     # queries must be 16-byte aligned (TMA)

    # the BM25 select stage on caller-owned candidate lists: workspace 2 * Q * ceil(m / 4096) * k elements
    def bsel(Q=3, m=5000, k=10, ws_elems=2 * 3 * 2 * 10, **kw):
        a = dict(scores=p, idx=p, ws_s=p, ws_i=p, out_s=p, out_i=p)
        a.update(kw)
        return l.rmu_debug_bm25_select(a["scores"], a["idx"], Q, m, k, a["ws_s"], a["ws_i"], ws_elems, a["out_s"],
                                       a["out_i"], None)

    assert bsel(k=0) == -3 and bsel(k=257) == -3 and bsel(k=-1) == -3
    assert bsel(Q=65536, ws_elems=1 << 40) == -3 and b"rmu_debug_bm25_select" in l.rmu_last_error()
    assert bsel(Q=0) == -1 and bsel(Q=-2) == -1 and bsel(m=0) == -1 and bsel(m=-4096) == -1
    for name in ("scores", "idx", "ws_s", "ws_i", "out_s", "out_i"):
        assert bsel(**{name: None}) == -1, name
    assert bsel(ws_elems=2 * 3 * 2 * 10 - 1) == -1                      # one element short
    assert bsel(m=4096, ws_elems=2 * 3 * 10 - 1) == -1 and bsel(m=4097, ws_elems=2 * 3 * 2 * 10 - 1) == -1
    assert bsel(Q=65535, m=1, k=256, ws_elems=2 * 65535 * 256 - 1) == -1

    # the KV-cache append: rows pos0 .. pos0 + T - 1 of a cache of cap rows
    def kva(T=4, heads=8, kv_heads=2, pos0=0, cap=16, **kw):
        a = dict(hi=p, lo=p, kv=p)
        a.update(kw)
        return l.rmu_debug_kv_append(a["hi"], a["lo"], T, heads, kv_heads, pos0, cap, a["kv"], None)

    for name in ("hi", "lo", "kv"):
        assert kva(**{name: None}) == -1, name
    for name in ("T", "heads", "kv_heads"):
        assert kva(**{name: 0}) == -1 and kva(**{name: -1}) == -1, name
    assert kva(pos0=-1) == -1 and b"rmu_debug_kv_append" in l.rmu_last_error()
    assert kva(pos0=13) == -1 and kva(T=17) == -1 and kva(cap=0) == -1          # pos0 + T > cap
    assert kva(T=1, pos0=2 ** 31 - 1, cap=2 ** 31 - 1) == -1                    # pos0 + T overflows int32
    assert kva(heads=6, kv_heads=4) == -3 and kva(heads=3, kv_heads=2) == -3    # heads % kv_heads

    # the q / k step: q_norm and k_norm both null (Llama) or both set; one of them alone is refused
    def qk(qn=p, kn=p, T=3, heads=8, kv=2, rows=16, **kw):
        a = dict(x=p, pos=p, cos=p, sin=p, hi=p, lo=p)
        a.update(kw)
        return l.rmu_debug_qk_norm_rope(a["x"], T, heads, kv, a["pos"], qn, kn, 1e-6, 1.0, a["cos"], a["sin"], rows,
                                        a["hi"], a["lo"], None, None)

    assert qk(qn=None) == -1 and qk(kn=None) == -1 and b"rmu_debug_qk_norm_rope" in l.rmu_last_error()
    for norms in ((p, p), (None, None)):
        for name in ("x", "pos", "cos", "sin", "hi", "lo"):
            assert qk(*norms, **{name: None}) == -1, name
        assert qk(*norms, T=0) == -1 and qk(*norms, heads=0) == -1 and qk(*norms, kv=0) == -1
        assert qk(*norms, rows=0) == -1


def test_encoder_create_refuses_weights_the_split_planes_cannot_hold(built_lib):
    """GEMM weights travel as fp16 planes, and fp16 rounds |w| >= 65520 to inf: rmu_encoder_create refuses such a
    weight on the host, before any CUDA call.  Tables, biases, LayerNorm parameters and the head stay fp32."""
    from ragmeup_b200 import _lib
    from ragmeup_b200.weights import PRESETS, synthetic_bert_weights, weight_names
    l = _lib.lib()
    cfg = PRESETS["tiny"][0]
    names = [n for n, _ in weight_names(cfg, True)]
    base = synthetic_bert_weights(cfg, seed=0, with_head=True)

    def create(name, idx, value):
        w = {k: v.copy() for k, v in base.items()}
        w[name].reshape(-1)[idx] = value
        arrs = [np.ascontiguousarray(w[n]) for n in names]
        ptrs = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        cc = _lib.BertConfigC(cfg.vocab_size, cfg.hidden, cfg.layers, cfg.heads, cfg.ffn, cfg.max_pos, cfg.type_vocab,
                              cfg.num_labels, cfg.ln_eps)
        h = ctypes.c_void_p()
        rc = l.rmu_encoder_create(ctypes.byref(cc), ptrs, len(arrs), 1, ctypes.byref(h))
        if rc == 0:
            l.rmu_encoder_destroy(h)
        return rc

    for name in ("encoder.layer.1.intermediate.dense.weight", "encoder.layer.0.attention.self.query.weight",
                 "encoder.layer.0.attention.self.value.weight", "encoder.layer.1.attention.output.dense.weight",
                 "encoder.layer.0.output.dense.weight", "encoder.layer.1.attention.self.key.weight"):
        for v in (7e4, -7e4, 65520.0, np.inf, -np.inf):
            assert create(name, 37, v) == -3, (name, v)
        assert b"65520" in l.rmu_last_error()
        # 65 519 (and 65 519.996, which rounds hi to 65 504) pass the check: without a device the next step fails
        for v in (65519.0, float(np.nextafter(np.float32(65520), np.float32(0))), -65519.0):
            assert create(name, 37, v) in (0, -2), (name, v)
    for name in ("embeddings.word_embeddings.weight", "encoder.layer.0.attention.self.query.bias",
                 "encoder.layer.0.output.LayerNorm.weight", "pooler.dense.weight", "classifier.weight"):
        assert create(name, 0, 7e4) in (0, -2), name


def test_encoder_refuses_a_batch_without_tokens(built_lib):
    """Empty sequences are allowed, but a batch of empty sequences only (total_tokens = 0), or no sequence at all, is
    refused with RMU_ERR_ARG before the handle is read or any CUDA call is made (include/ragmeup_b200.h)"""
    from ragmeup_b200 import _lib
    l = _lib.lib()
    p = 1 << 20
    fake = ctypes.c_void_p(p)                               # never dereferenced: every call below is refused first
    for B, T in ((3, 0), (1, 0), (0, 0), (0, 5), (-1, 5), (3, -1)):
        assert l.rmu_encoder_embed(fake, p, None, p, B, T, 1, 0, 1, p, None) == -1, (B, T)
        assert l.rmu_encoder_classify(fake, p, None, p, B, T, 1, p, None) == -1, (B, T)
        assert l.rmu_encoder_hidden(fake, p, p, p, B, T, 1, p, None) == -1, (B, T)
        assert l.rmu_encoder_embed_host(fake, p, None, p, B, T, 1, 1, 0, p, None) == -1, (B, T)
        assert l.rmu_encoder_classify_host(fake, p, p, p, B, T, 1, p, None) == -1, (B, T)
    assert b"encoder" in l.rmu_last_error()


def test_product_fails_loudly_without_cuda(built_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from ragmeup_b200 import _lib
    from ragmeup_b200.index import FlatIndex
    with pytest.raises(_lib.RmuError):
        FlatIndex(384, "l2")
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    with pytest.raises(_lib.RmuError):
        HuggingFaceEmbeddings(model_name="synthetic:tiny", model_kwargs={"device": "cpu"})
    with pytest.raises(_lib.RmuError):
        HuggingFaceEmbeddings(model_name="synthetic:tiny", model_kwargs={"device": "cuda"})


def test_product_never_imports_oracle():
    """the oracle is test infrastructure: no product module may import it"""
    pkg = os.path.join(ROOT, "ragmeup_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
