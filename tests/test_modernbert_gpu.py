"""ModernBERT on the GPU encoder: the three E1 epilogues (rotary q / k, GeGLU, fp32 residual), E2's sliding window, the
head, the whole pre-LN stack against the float64 forward, and the product classes."""
from __future__ import annotations

import json
import math
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import encoder_kernels_ref as ref
from oracle import modernbert_ref as mr
from ragmeup_b200.documents import Document
from ragmeup_b200.weights import PRESETS, ModernBertConfig, rope_tables, synthetic_bert_weights

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
C_ATT = 8.0                    # as test_deberta_gpu.py: |err| <= 8 * 2^-22 * max|V| * (1 + A)
SYL = ["ba", "ce", "di", "fo", "gu", "ha", "je", "ki", "lo", "mu", "na", "pe", "qi", "ro", "su", "ta"]


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def _cfg(preset):
    return ModernBertConfig(**asdict(PRESETS[preset][0]))


def _texts(n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    return [" ".join("".join(SYL[j] for j in rng.integers(0, len(SYL), rng.integers(1, 4)))
                     for _ in range(int(rng.integers(lo, hi + 1)))) for _ in range(n)]


def _planes(x):
    return [torch.from_numpy(p).cuda() for p in ref.split_f16(np.ascontiguousarray(x, dtype=np.float32))]


def _j(p):
    return p[0].double() + p[1].double()


def _gemm_ex(mode, a, wp, M, N, K, bias, res=None, qcols=0, qscale=1.0, pos=None, tabs=(None, None), rows=0, hd=64,
             out_f32=None, out_cols=None):
    L = _lib()
    oh = ol = None
    if out_f32 is None:
        oh = torch.full((M, out_cols or N), float("nan"), dtype=torch.float16, device="cuda")
        ol = torch.full_like(oh, float("nan"))
    L.check(L.lib().rmu_debug_gemm_ex(mode, _ptr(a[0]), _ptr(a[1]), M, _ptr(wp[0]), _ptr(wp[1]), M, N, K, _ptr(bias),
                                      _ptr(res), qcols, qscale, _ptr(pos), _ptr(tabs[0]), _ptr(tabs[1]), rows, hd, 0,
                                      _ptr(out_f32), _ptr(oh), _ptr(ol), L.stream_ptr()), f"rmu_debug_gemm_ex {mode}")
    torch.cuda.synchronize()
    return out_f32.double() if out_f32 is not None else oh.double() + ol.double()


# ------------------------------------------------------------------------------------------------- E1
@pytest.mark.parametrize("H,heads", [(768, 12), (256, 8)])
def test_rope_epilogue_matches_float64(cuda, H, heads):
    """q and k rotated at positions up to 8191 with both theta tables, v untouched, q scaled; against float64 on the
    split operands with the same float32 tables"""
    d = H // heads
    cfg = ModernBertConfig(hidden=H, heads=heads, layers=1, ffn=128, max_pos=8192)
    cg, sg, cl, sl = [torch.from_numpy(t).cuda() for t in rope_tables(cfg)]
    rng = np.random.default_rng(1)
    M, K, N = 600, 128, 3 * H
    pos = rng.integers(0, 8192, M).astype(np.int32)
    pos[:4] = [0, 1, 8190, 8191]
    a = _planes(rng.standard_normal((M, K)))
    wp = _planes(rng.standard_normal((N, K)) * 0.1)
    bias = torch.from_numpy(rng.standard_normal(N).astype(np.float32) * 0.1).cuda()
    pos_d = torch.from_numpy(pos).cuda()
    qs = math.log2(math.e) / math.sqrt(d)
    A, Wt = _j(a), _j(wp)
    raw = A @ Wt.t() + bias.double()
    mag = (A.abs() @ Wt.abs().t() + bias.double().abs())
    for tabs in ((cg, sg), (cl, sl)):
        got = _gemm_ex(4, a, wp, M, N, K, bias, qcols=H, qscale=qs, pos=pos_d, tabs=tabs, rows=8192, hd=d)
        want = raw.clone()
        bound = mag.clone()
        c, s = tabs[0].double()[pos_d.long()], tabs[1].double()[pos_d.long()]
        for part in (0, 1):
            x = want[:, part * H:(part + 1) * H].reshape(M, heads, d)
            xb = bound[:, part * H:(part + 1) * H].reshape(M, heads, d)
            rot = mr.rotate(x.transpose(0, 1), c, s).transpose(0, 1)
            want[:, part * H:(part + 1) * H] = rot.reshape(M, H)
            bsum = xb[..., :d // 2] + xb[..., d // 2:]
            bound[:, part * H:(part + 1) * H] = torch.cat([bsum, bsum], -1).reshape(M, H)
        want[:, :H] *= qs
        bound[:, :H] *= qs
        ratio = float(((got - want).abs() / (16 * 2.0 ** -22 * bound)).max())
        print(f"\nrope H={H}: max |err| / bound = {ratio:.3g}")
        assert torch.isfinite(got).all() and ratio <= 1.0
        assert float((raw[:, :2 * H] - want[:, :2 * H]).abs().max()) > 1.0        # the rotation is there
        assert torch.equal(want[:, 2 * H:], raw[:, 2 * H:])


def _geglu_rows(x, F):
    """the reorder rmu_encoder_create_modernbert applies to Wi / bi: 128-row blocks of 64 input | 64 gate rows"""
    out = np.empty_like(x)
    for k in range(F // 64):
        out[128 * k:128 * k + 64] = x[64 * k:64 * k + 64]
        out[128 * k + 64:128 * k + 128] = x[F + 64 * k:F + 64 * k + 64]
    return out


def test_geglu_epilogue_matches_float64(cuda):
    """gelu(in + b_in) * (gate + b_gate) at ModernBERT-large's F = 2624 (not a multiple of 128): N = 2 F"""
    rng = np.random.default_rng(2)
    M, K, F = 300, 128, 2624
    a = _planes(rng.standard_normal((M, K)))
    wnat = (rng.standard_normal((2 * F, K)) * 0.1).astype(np.float32)
    bnat = (rng.standard_normal(2 * F) * 0.5).astype(np.float32)
    wp = _planes(_geglu_rows(wnat, F))
    bias = torch.from_numpy(_geglu_rows(bnat[:, None], F)[:, 0].copy()).cuda()
    got = _gemm_ex(5, a, wp, M, 2 * F, K, bias, out_cols=F)
    A = _j(a)
    Wn = _j(_planes(wnat))
    h = A @ Wn.t() + torch.from_numpy(bnat).double().cuda()
    mag = A.abs() @ Wn.abs().t() + torch.from_numpy(np.abs(bnat)).double().cuda()
    xin, gate = h[:, :F], h[:, F:]
    want = mr._gelu(xin) * gate
    # |gelu'| <= 1.13; the erf approximation adds 1.5e-7 |x| / 2 per GELU
    bound = 16 * 2.0 ** -22 * (1.13 * mag[:, :F] * gate.abs() + (xin.abs() + mag[:, :F]) * mag[:, F:]) \
        + 1e-7 * xin.abs() * gate.abs() + 2.0 ** -22 * want.abs()
    ratio = float(((got - want).abs() / bound).max())
    print(f"\ngeglu: max |err| / bound = {ratio:.3g}")
    assert torch.isfinite(got).all() and ratio <= 1.0
    assert float((mr._gelu(gate) * xin - want).abs().max()) > 100 * float((got - want).abs().max())


def test_fp32_residual_epilogue_in_place(cuda):
    """out = A W^T + b + res with out and res the same array, residual values far outside fp16's range"""
    rng = np.random.default_rng(3)
    M, K, N = 333, 2624, 768
    a = _planes(rng.standard_normal((M, K)))
    wp = _planes(rng.standard_normal((N, K)) * 0.05)
    bias = torch.from_numpy(rng.standard_normal(N).astype(np.float32)).cuda()
    res = torch.from_numpy((rng.standard_normal((M, N)) * 1e5).astype(np.float32)).cuda()
    res0 = res.double().clone()
    got = _gemm_ex(6, a, wp, M, N, K, bias, res=res, out_f32=res)
    A, Wt = _j(a), _j(wp)
    want = A @ Wt.t() + bias.double() + res0
    bound = 16 * 2.0 ** -22 * (A.abs() @ Wt.abs().t() + bias.double().abs()) + 2.0 ** -23 * want.abs()
    ratio = float(((got - want).abs() / bound).max())
    print(f"\nresidual in place: max |err| / bound = {ratio:.3g}")
    assert torch.isfinite(got).all() and ratio <= 1.0


# ------------------------------------------------------------------------------------------------- E2 window
def _first_block_masked_rows(lens, w, nw=10):
    """rows whose first key block the kernel computes holds no visible key (the running max is still -inf there)"""
    n = 0
    for S in lens:
        for rbase in range(0, S, 16 * nw):
            k0, k1 = max(0, rbase - w), min(S, rbase + 16 * nw + w)
            for r0 in range(rbase, min(S, rbase + 16 * nw), 16):
                blocks = [j0 for j0 in range(k0, k1, 32) if not (j0 + 31 < r0 - w or j0 > r0 + 15 + w)]
                for i in range(r0, min(S, r0 + 16)):
                    j0 = blocks[0]
                    if all(abs(i - j) > w for j in range(j0, min(j0 + 32, k1))):
                        n += 1
    return n


@pytest.mark.parametrize("H,heads,window", [(768, 12, 64), (768, 12, 16), (768, 12, 20), (256, 8, 16), (256, 8, 20)])
def test_attention_window_matches_float64(cuda, H, heads, window):
    """lengths across the window (65, 66, 129), the 160-row CTA edge (160, 161), a key super-block (257) and long rows
    (600, 1000), several sequences per batch, at d_h 64 and 32.  With a half-window that is not a multiple of 16 (20),
    rows near the start of a sequence meet a key block that is fully masked for them before any visible key (the -inf
    max guard)"""
    lens = [1, 2, 65, 66, 129, 160, 161, 257, 600, 1000]
    if window % 16:
        assert _first_block_masked_rows(lens, window) > 0
    rng = np.random.default_rng(4)
    T = sum(lens)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    qs = math.log2(math.e) / 8
    x = rng.standard_normal((T, 3 * H)).astype(np.float32)
    x[:, :H] *= 0.6 * qs * 8
    qkv = _planes(x)
    cu_d = torch.from_numpy(cu).cuda()
    ch = torch.full((T, H), float("nan"), dtype=torch.float16, device="cuda")
    cl = torch.full_like(ch, float("nan"))
    L = _lib()
    L.check(L.lib().rmu_debug_attention_window(_ptr(qkv[0]), _ptr(qkv[1]), _ptr(cu_d), len(lens), H, heads, max(lens),
                                               window, _ptr(ch), _ptr(cl), L.stream_ptr()), "rmu_debug_attention_window")
    torch.cuda.synchronize()
    got = ch.double() + cl.double()
    want = mr.window_attention_ref(_j(qkv), cu, heads, window)
    vmax = float(_j(qkv)[:, 2 * H:].abs().max())
    err = float((got - want).abs().max())
    assert torch.isfinite(got).all()
    assert err <= C_ATT * 2.0 ** -22 * vmax * 32, (err, vmax)
    assert float((want - mr.window_attention_ref(_j(qkv), cu, heads, 0)).abs().max()) > 100 * err


@pytest.mark.parametrize("H,heads", [(768, 12), (256, 8)])
def test_attention_wide_window_is_plain_attention(cuda, H, heads):
    """with window >= S - 1 the windowed kernel stages the keys of the plain one in the same order: bit-identical"""
    lens = [3, 161, 320, 77, 500]
    rng = np.random.default_rng(6)
    T = sum(lens)
    cu_d = torch.from_numpy(np.r_[0, np.cumsum(lens)].astype(np.int32)).cuda()
    x = rng.standard_normal((T, 3 * H)).astype(np.float32)
    x[:, :H] *= 0.4
    qkv = _planes(x)
    L = _lib()
    outs = []
    for win in (None, max(lens) - 1, 10 ** 6):
        ch = torch.full((T, H), float("nan"), dtype=torch.float16, device="cuda")
        cl = torch.full_like(ch, float("nan"))
        if win is None:
            rc = L.lib().rmu_debug_attention(_ptr(qkv[0]), _ptr(qkv[1]), _ptr(cu_d), len(lens), H, heads, max(lens), 10,
                                             _ptr(ch), _ptr(cl), L.stream_ptr())
        else:
            rc = L.lib().rmu_debug_attention_window(_ptr(qkv[0]), _ptr(qkv[1]), _ptr(cu_d), len(lens), H, heads, max(lens),
                                                    win, _ptr(ch), _ptr(cl), L.stream_ptr())
        L.check(rc, "attention")
        torch.cuda.synchronize()
        outs.append((ch.clone(), cl.clone()))
    for o in outs[1:]:
        assert torch.equal(o[0].view(torch.int16), outs[0][0].view(torch.int16))
        assert torch.equal(o[1].view(torch.int16), outs[0][1].view(torch.int16))


# ------------------------------------------------------------------------------------------------- head
@pytest.mark.parametrize("mode", [0, 1])
def test_head_matches_float64(cuda, mode):
    """pool_kernel (mean or CLS, not normalised) then the head, against float64"""
    rng = np.random.default_rng(7)
    H, nl = 768, 2
    lens = [1, 7, 130, 64]
    T = sum(lens)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    hp = _planes(rng.standard_normal((T, H)) * 3)
    head = {"head.dense.weight": rng.standard_normal((H, H)) * 0.05, "head.dense.bias": rng.standard_normal(H) * 0.1,
            "head.norm.weight": 1 + 0.1 * rng.standard_normal(H), "head.norm.bias": 0.1 * rng.standard_normal(H),
            "classifier.weight": rng.standard_normal((nl, H)) * 0.1, "classifier.bias": rng.standard_normal(nl)}
    hd = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in head.items()}
    L = _lib()
    cu_d = torch.from_numpy(cu).cuda()
    pooled = torch.empty((len(lens), H), dtype=torch.float32, device="cuda")
    L.check(L.lib().rmu_debug_pool(_ptr(hp[0]), _ptr(hp[1]), _ptr(cu_d), len(lens), H, mode, 0, _ptr(pooled),
                                   L.stream_ptr()), "pool")
    out = torch.empty((len(lens), nl), dtype=torch.float32, device="cuda")
    L.check(L.lib().rmu_debug_modernbert_head(_ptr(pooled), len(lens), H, nl, _ptr(hd["head.dense.weight"]),
                                              _ptr(hd["head.dense.bias"]), _ptr(hd["head.norm.weight"]),
                                              _ptr(hd["head.norm.bias"]), 1e-5, _ptr(hd["classifier.weight"]),
                                              _ptr(hd["classifier.bias"]), _ptr(out), L.stream_ptr()), "head")
    torch.cuda.synchronize()
    h = _j(hp)
    p = torch.stack([h[cu[b]] if mode == 1 else h[cu[b]:cu[b + 1]].mean(0) for b in range(len(lens))])
    V = {k: v.double() for k, v in hd.items()}
    y = mr._ln(mr._gelu(p @ V["head.dense.weight"].t() + V["head.dense.bias"]), V["head.norm.weight"],
               V["head.norm.bias"], 1e-5)
    want = y @ V["classifier.weight"].t() + V["classifier.bias"]
    err = float((out.double() - want).abs().max())
    print(f"\nhead mode {mode}: max |err| = {err:.3g}")
    assert err < 1e-4 * max(1.0, float(want.abs().max()))


# ------------------------------------------------------------------------------------------------- whole stack
# The rule of test_deberta_gpu.py: against the float64 forward on the split weights, the GPU's max and rms error stay
# within c x those of the fp32 forward on the same weights + FLOOR u |ref|.  Measured on an H100 (max / rms): tiny x4
# 4.0 / 3.3 on the hidden state, 5.4 / 5.4 on the logits; tiny-window 1.2 / 1.3 and 3.7 / 4.2; base 8.4 / 10.5 and
# 19 / 24.5 (bge-reranker-base's XLM-R stack: 23).  c is about twice the largest of its case.  Empty sequences (length
# 0) pool to a zero vector and go through the head like any other row.
FLOOR = 4.0
STACK = {
    "tiny-modernbert x4": ("tiny-modernbert", 3, 4.0, [1, 2, 0, 65, 66, 129, 161, 700, 0], 12),
    "tiny-modernbert-window": ("tiny-modernbert-window", 0, 1.0, [5, 33, 65, 0, 161, 600], 10),
    "modernbert-base": ("modernbert-base", 1, 1.0, [65, 0, 129, 161, 640], 50),
}


@pytest.mark.parametrize("case", list(STACK))
def test_modernbert_stack_matches_float64_forward(cuda, case):
    from ragmeup_b200.encoder import BertEncoder
    preset, seed, scale, lens, c = STACK[case]
    cfg = _cfg(preset)
    w = synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale)
    enc = BertEncoder(cfg, w, with_head=True)
    wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    w32 = {k: ref.split_weight(v).float() if k.endswith(mr.GEMM) else v for k, v in wd.items()}
    rng = np.random.default_rng(seed)
    ids = np.concatenate([rng.integers(3, cfg.vocab_size, n) for n in lens]).astype(np.int32)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    mx = max(lens)
    got = {"hidden": enc.hidden_tokens(ids, None, cu, mx).double(), "logits": enc.classify_tokens(ids, None, cu, mx)}
    want = mr.modernbert_stack(wd, cfg, ids, cu, torch.float64, "split", device="cuda")
    f32 = mr.modernbert_stack(w32, cfg, ids, cu, torch.float32, "fp32", device="cuda")
    report, fails = [], []
    for name in ("hidden", "logits"):
        g, w_, f = got[name].double(), want[name], f32[name].double()
        assert torch.isfinite(g).all(), name
        d, e = (g - w_).abs(), (f - w_).abs()
        gmax, grms, fmax, frms = float(d.max()), float(d.pow(2).mean().sqrt()), float(e.max()), float(e.pow(2).mean().sqrt())
        mag_max, mag_rms = float(w_.abs().max()), float(w_.pow(2).mean().sqrt())
        report.append(f"{name} max {gmax:.3g} / fp32 {fmax:.3g} = {gmax / fmax:.3g}, rms {grms:.3g} / {frms:.3g} = "
                      f"{grms / frms:.3g}")
        if gmax > c * fmax + FLOOR * U * mag_max or grms > c * frms + FLOOR * U * mag_rms:
            fails.append(report[-1])
    print(f"\nModernBERT stack {case}:\n  " + "\n  ".join(report))
    assert not fails, f"{case}: beyond {c} x fp32's error: " + "; ".join(fails)
    assert np.array_equal(enc.classify_host(ids, None, cu), got["logits"].cpu().numpy())
    # the embedder's pooling reads the same hidden state
    for pooling in ("cls", "mean"):
        e = enc.embed_tokens(ids, None, cu, mx, pooling, False).double()
        p = torch.stack([torch.zeros(cfg.hidden, dtype=torch.float64, device="cuda") if n == 0
                         else got["hidden"][cu[b]] if pooling == "cls" else got["hidden"][cu[b]:cu[b + 1]].mean(0)
                         for b, n in enumerate(lens)])
        assert float((e - p).abs().max()) <= 1e-5 * float(p.abs().max())


@pytest.mark.parametrize("case", range(4))
def test_golden_logits(cuda, golden_dir, case):
    """transformers' ModernBertForSequenceClassification (tests/golden/modernbert.npz) from the encoder: logits, and the
    final hidden state's first, last and mean rows, within 1e-3"""
    import importlib.util
    import os
    from ragmeup_b200.encoder import BertEncoder
    spec = importlib.util.spec_from_file_location("make_golden_modernbert",
                                                  os.path.join(golden_dir, "make_golden_modernbert.py"))
    gm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gm)
    preset, seed, scale, pooling, lens = gm.CASES[case]
    g = np.load(f"{golden_dir}/modernbert.npz")
    key = gm.case_key(preset, seed, scale, pooling)
    cfg = gm.case_config(preset, pooling)
    enc = BertEncoder(cfg, synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale), with_head=True)
    assert g[key + "_mask"].sum(1).tolist() == lens
    ids = np.concatenate([g[key + "_ids"][b, :n] for b, n in enumerate(lens)]).astype(np.int32)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    got = enc.classify_host(ids, None, cu)
    want = g[key + "_logits"]
    assert np.abs(got - want).max() < 1e-3 * max(1.0, float(np.abs(want).max()))
    h = enc.hidden_tokens(ids, None, cu, max(lens)).cpu().numpy()
    assert np.abs(h[cu[:-1]] - g[key + "_h_first"]).max() < 1e-3
    assert np.abs(h[cu[1:] - 1] - g[key + "_h_last"]).max() < 1e-3
    mean = np.stack([h[cu[b]:cu[b + 1]].mean(0) for b in range(len(lens))])
    assert np.abs(mean - g[key + "_h_mean"]).max() < 1e-3


def test_sequence_past_max_pos_is_refused(cuda):
    from ragmeup_b200 import _lib as L
    from ragmeup_b200.encoder import BertEncoder
    cfg = _cfg("tiny-modernbert")
    enc = BertEncoder(cfg, synthetic_bert_weights(cfg, seed=0, with_head=True), with_head=True)
    n = cfg.max_pos + 1
    with pytest.raises(L.RmuError, match="max_position_embeddings"):
        enc.classify_host(np.full(n, 5, np.int32), None, np.array([0, n], np.int32))
    enc.classify_host(np.full(n - 1, 5, np.int32), None, np.array([0, n - 1], np.int32))


# ------------------------------------------------------------------------------------------------- product
@pytest.fixture(scope="module")
def reranker():
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.weights import resolve_model
    name = "synthetic:tiny-modernbert:2:4.0"
    ce = HuggingFaceCrossEncoder(model_name=name)
    cfg, w, *_ = resolve_model(name, with_head=True)
    return ce, w, cfg


def _oracle_scores(ce, w, cfg, pairs):
    ids, _typ, cu = ce._pairs([p[0].strip() for p in pairs], [p[1].strip() for p in pairs])
    logits = mr.modernbert_stack(w, cfg, ids, cu, torch.float32, device="cuda")["logits"]
    return torch.sigmoid(logits)[:, 0].cpu().numpy()


def test_score_matches_fp32_oracle(reranker):
    """RAGMeUp's call (1 query, 14 documents) and a pair past 600 tokens, against the fp32 oracle"""
    ce, w, cfg = reranker
    assert ce.activation == "sigmoid" and ce.max_length == cfg.max_pos and not ce._types
    q = _texts(1, 6, 12, 1)[0]
    docs = _texts(13, 60, 120, 2) + _texts(1, 500, 700, 3)
    pairs = [(q, d) for d in docs]
    got = ce.score(pairs)
    assert got.dtype == np.float32 and got.shape == (14,)
    assert np.abs(got - _oracle_scores(ce, w, cfg, pairs)).max() < 1e-3
    assert np.abs(ce.score_tensor(pairs).cpu().numpy() - got).max() <= 1e-6


def test_embeddings_match_fp32_oracle(cuda):
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.weights import resolve_model
    name = "synthetic:tiny-modernbert-window:5"
    emb = HuggingFaceEmbeddings(model_name=name)
    cfg, w, *_ = resolve_model(name, with_head=False)
    texts = _texts(9, 3, 200, 8)
    got = np.asarray(emb.embed_documents(texts), dtype=np.float32)
    ids, _typ, cu = emb._ragged(texts)
    h = mr.modernbert_stack(w, cfg, ids, cu, torch.float32, device="cuda")["hidden"]
    want = torch.stack([h[cu[b]:cu[b + 1]].mean(0) for b in range(len(texts))])
    want = torch.nn.functional.normalize(want, dim=-1).cpu().numpy()
    assert np.abs(got - want).max() < 1e-4
    t = emb.encode_tensor(texts).cpu().numpy()
    assert np.abs(t - got).max() <= 1e-6


def test_snapshot_loads_and_scores(cuda, tmp_path):
    """a tiny ModernBertForSequenceClassification saved with save_pretrained, its config.json rewritten in the release
    form, and a tokenizer.json: HuggingFaceCrossEncoder scores as transformers does (eager attention, fp32)"""
    transformers = pytest.importorskip("transformers")
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.tokenizer import build_wordpiece, synthetic_vocab
    vocab = synthetic_vocab(1000)
    hc = transformers.ModernBertConfig(
        vocab_size=1000, hidden_size=128, num_hidden_layers=4, num_attention_heads=2, intermediate_size=192,
        max_position_embeddings=1024, local_attention=32, global_attn_every_n_layers=3, classifier_pooling="mean",
        pad_token_id=vocab["[PAD]"], bos_token_id=vocab["[CLS]"], eos_token_id=vocab["[SEP]"],
        cls_token_id=vocab["[CLS]"], sep_token_id=vocab["[SEP]"], num_labels=1)
    torch.manual_seed(0)
    model = transformers.ModernBertForSequenceClassification(hc).eval()
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "norm" not in n:
                p.normal_(0.0, 0.08)
    model.save_pretrained(tmp_path, safe_serialization=True)
    cfgd = json.loads((tmp_path / "config.json").read_text())
    for k in ("layer_types", "rope_parameters"):
        cfgd.pop(k, None)
    cfgd.update(global_attn_every_n_layers=3, global_rope_theta=160000.0, local_rope_theta=10000.0, local_attention=32)
    (tmp_path / "config.json").write_text(json.dumps(cfgd))
    tok = build_wordpiece(vocab)
    tok.save(str(tmp_path / "tokenizer.json"))
    ce = HuggingFaceCrossEncoder(model_name=str(tmp_path))
    assert ce.config.layer_windows == (0, 16, 16, 0) and ce.config.classifier_pooling == "mean"
    pairs = [(q, d) for q in _texts(2, 4, 8, 9) for d in _texts(5, 20, 150, 10)]
    got = ce.score(pairs)
    ids, _typ, cu = ce._pairs([p[0] for p in pairs], [p[1] for p in pairs])
    ref_model = transformers.ModernBertForSequenceClassification.from_pretrained(tmp_path, attn_implementation="eager")
    want = []
    with torch.no_grad():
        for b in range(len(pairs)):
            x = torch.from_numpy(ids[cu[b]:cu[b + 1]].astype(np.int64))[None]
            want.append(float(torch.sigmoid(ref_model.eval()(x).logits)[0, 0]))
    assert np.abs(got - np.asarray(want, np.float32)).max() < 1e-3


def test_mmr_then_modernbert_rerank(reranker):
    """Milvus MMR retrieval, then ScoredCrossEncoderReranker with the ModernBERT reranker"""
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.reranker import ScoredCrossEncoderReranker
    from ragmeup_b200.vectorstore import Milvus
    ce, w, cfg = reranker
    emb = HuggingFaceEmbeddings(model_name="synthetic:tiny-modernbert")
    docs = _texts(200, 20, 60, 6)
    db = Milvus.from_documents([], emb, drop_old=True, connection_args={"uri": "data.db"}, collection_name="modernbert")
    db.add_documents([Document(t, {"id": f"id{i}"}) for i, t in enumerate(docs)], ids=[f"id{i}" for i in range(200)])
    retriever = db.as_retriever(search_type="mmr", search_kwargs={"k": 10})
    rr = ScoredCrossEncoderReranker(model=ce, top_n=3)
    for qtext in _texts(3, 5, 12, 7):
        found = retriever.invoke(qtext)
        assert len(found) == 10
        top = rr.compress_documents(found, qtext)
        pairs = [(qtext, d.page_content) for d in found]
        got = ce.score(pairs)
        order = sorted(range(len(found)), key=lambda i: got[i], reverse=True)[:3]
        assert [d.page_content for d in top] == [found[i].page_content for i in order]
        assert [d.metadata["relevance_score"] for d in top] == [got[i] for i in order]
        assert np.abs(got - _oracle_scores(ce, w, cfg, pairs)).max() < 1e-3
