"""CPU: the float64 per-kernel references (oracle/encoder_kernels_ref.py) against independent restatements, so that
tests/test_encoder_kernels_gpu.py judges the kernels against something that is itself pinned."""
import math
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import bert_ref
from oracle import encoder_kernels_ref as ref
from ragmeup_b200.weights import PRESETS, BertConfig, synthetic_bert_weights


def test_split_emulation_matches_torch_half():
    rng = np.random.default_rng(0)
    # normal range, the subnormal lo range (|v| < ~0.125), hi itself subnormal, exact fp16 values, signed zero
    v = np.concatenate([rng.standard_normal(4096) * s for s in (1e-6, 1e-4, 1e-3, 0.05, 1.0, 16.0, 3e3)]
                       + [np.array([0.0, -0.0, 1.0, -2.5, 65504.0, 6.1e-5, 2.0 ** -24, 2.0 ** -25])]).astype(np.float32)
    hi, lo = ref.split_f16(v)
    t = torch.from_numpy(v)
    th = t.half()
    tl = (t - th.float()).half()
    assert np.array_equal(hi.view(np.uint16), th.numpy().view(np.uint16))
    assert np.array_equal(lo.view(np.uint16), tl.numpy().view(np.uint16))
    assert (np.abs(lo[np.abs(v) < 0.06]) < 2.0 ** -14).any()       # the subnormal lo range is exercised
    # round-to-nearest in order: |lo| <= half an fp16 ulp of hi
    assert (np.abs(lo.astype(np.float64)) <= 0.5 * ref.ulp_f16(hi)).all()


def test_attention_reference_is_the_softmax_when_q_carries_log2e():
    rng = np.random.default_rng(1)
    heads, dh = 3, 32
    H = heads * dh
    lens = [1, 17, 40]
    cu = np.r_[0, np.cumsum(lens)]
    T = cu[-1]
    q, k, v = (rng.standard_normal((T, H)) for _ in range(3))
    scale = 1.0 / math.sqrt(dh)
    qkv = np.concatenate([q * scale * math.log2(math.e), k, v], 1).astype(np.float32)
    hi, lo = ref.split_f16(qkv)
    ctx, A = ref.attention_ref(hi, lo, cu, heads)
    x = torch.from_numpy(ref.join(hi, lo))
    qq, kk, vv = x[:, :H] / math.log2(math.e), x[:, H:2 * H], x[:, 2 * H:]     # the unscaled-by-log2e q of the planes
    for b in range(len(lens)):
        s = slice(cu[b], cu[b + 1])
        for h in range(heads):
            d = slice(h * dh, (h + 1) * dh)
            want = torch.softmax(qq[s, d] @ kk[s, d].T, -1) @ vv[s, d]           # q already carries 1/sqrt(d)
            assert (ctx[s, d] - want).abs().max() < 1e-12
            assert torch.allclose(A[s, h], (qq[s, d].abs() @ kk[s, d].abs().T).amax(1) * math.log2(math.e))


def test_gemm_reference_with_zero_lo_is_the_float64_product():
    rng = np.random.default_rng(2)
    M, N, K = 37, 128, 192
    a = rng.standard_normal((M, K)).astype(np.float16)
    w = rng.standard_normal((N, K)).astype(np.float16)
    z = np.zeros_like
    bias = rng.standard_normal(N).astype(np.float32)
    want = a.astype(np.float64) @ w.astype(np.float64).T
    out, x, S = ref.gemm_ref(ref.GEMM_BIAS_F32, a, z(a), w, z(w), np.zeros(N, np.float32))
    assert np.array_equal(out.numpy(), want)
    assert np.allclose(S.numpy(), np.abs(a.astype(np.float64)) @ np.abs(w.astype(np.float64)).T, rtol=1e-15, atol=0)
    # epilogues
    out, x, _ = ref.gemm_ref(ref.GEMM_BIAS_GELU_SPLIT, a, z(a), w, z(w), bias)
    assert np.allclose(out.numpy(), bert_ref._gelu_erf(torch.from_numpy(want + bias)).numpy(), rtol=1e-12, atol=1e-12)
    assert np.allclose(out.numpy(), [[0.5 * t * (1 + math.erf(t / math.sqrt(2))) for t in r] for r in want + bias],
                       rtol=1e-14, atol=1e-15)
    r = rng.standard_normal((M, N)).astype(np.float32)
    rh, rl = ref.split_f16(r)
    out, _, _ = ref.gemm_ref(ref.GEMM_BIAS_RESID_F32, a, z(a), w, z(w), bias, rh, rl)
    assert np.allclose(out.numpy(), want + bias + rh.astype(np.float64) + rl.astype(np.float64), rtol=0, atol=1e-12)
    out, _, _ = ref.gemm_ref(ref.GEMM_BIAS_SPLIT_QSCALE, a, z(a), w, z(w), bias, qcols=40, qscale=0.25)
    out = out.numpy()
    assert np.array_equal(out[:, :40], (want + bias)[:, :40] * 0.25) and np.array_equal(out[:, 40:], (want + bias)[:, 40:])
    # the lo planes enter as al * wh + ah * wl, never al * wl
    al = np.full_like(a, 2.0 ** -12)
    wl = np.full_like(w, 2.0 ** -12)
    out, _, _ = ref.gemm_ref(ref.GEMM_BIAS_F32, a, al, w, wl, np.zeros(N, np.float32))
    a64, w64 = a.astype(np.float64), w.astype(np.float64)
    assert np.allclose(out.numpy(), want + 2.0 ** -12 * (a64.sum(1)[:, None] + w64.sum(1)[None, :]), rtol=0, atol=1e-12)


def _blocked_rows(first, second):
    """the gated modes' weight layout: 128-row blocks of 64 rows of `first` then the 64 matching rows of `second`"""
    out = np.empty((2 * first.shape[0],) + first.shape[1:], first.dtype)
    for k in range(first.shape[0] // 64):
        out[128 * k:128 * k + 64] = first[64 * k:64 * k + 64]
        out[128 * k + 64:128 * k + 128] = second[64 * k:64 * k + 64]
    return out


def _planes64(x):
    hi, lo = ref.split_f16(x)
    return hi, lo, torch.from_numpy(ref.join(hi, lo))


@pytest.mark.parametrize("head_dim,qcols,N", [(64, 128, 384), (32, 128, 384), (64, 192, 640)])
def test_gemm_reference_rope_mode_is_modernbert_rotate(head_dim, qcols, N):
    """mode 4 against modernbert_ref.rotate per head on x = A W^T + b, positions clamped into the tables, q scaled by
    float32(qscale), v untouched (columns past 3 qcols included)"""
    from oracle import modernbert_ref as mr
    from ragmeup_b200.weights import rope_table
    rng = np.random.default_rng(head_dim + qcols)
    M, K, rows = 9, 64, 50
    ah, al, A = _planes64(rng.standard_normal((M, K)))
    wh, wl, W = _planes64(0.1 * rng.standard_normal((N, K)))
    bias = rng.standard_normal(N).astype(np.float32)
    cos, sin = rope_table(10000.0, head_dim, rows)
    pos = np.array([0, 1, rows - 1, -3, rows, rows + 70, 7, 23, 49], np.int32)
    qs = 1.4426950408889634 / math.sqrt(head_dim)
    out, x, S = ref.gemm_ref(ref.GEMM_BIAS_SPLIT_ROPE, ah, al, wh, wl, bias, qcols=qcols, qscale=qs, pos=pos,
                             rope_cos=cos, rope_sin=sin, head_dim=head_dim)
    acc = A @ W.T - torch.from_numpy(ref.join(al, np.zeros_like(al))).double() @ torch.from_numpy(
        ref.join(wl, np.zeros_like(wl))).T                  # the kernel's three products: no al * wl
    xx = acc + torch.from_numpy(bias).double()
    assert torch.allclose(x, xx, rtol=1e-13, atol=1e-13)
    assert torch.allclose(S, A.abs() @ W.abs().T, rtol=1e-13, atol=0)
    pc = torch.from_numpy(np.clip(pos, 0, rows - 1)).long()
    c, s = torch.from_numpy(cos).double()[pc], torch.from_numpy(sin).double()[pc]
    want = xx.clone()
    for part in (0, 1):
        blk = xx[:, part * qcols:(part + 1) * qcols].reshape(M, qcols // head_dim, head_dim).transpose(0, 1)
        want[:, part * qcols:(part + 1) * qcols] = mr.rotate(blk, c, s).transpose(0, 1).reshape(M, qcols)
    want[:, :qcols] *= float(np.float32(qs))
    assert torch.allclose(out, want, rtol=1e-13, atol=1e-13)
    assert torch.equal(out[:, 2 * qcols:], x[:, 2 * qcols:])
    # the partner of a q / k column is the other half of its head; a v column is its own
    P = ref.rope_partner(x, qcols, head_dim)
    h = head_dim // 2
    assert torch.equal(P[:, 0], x[:, h]) and torch.equal(P[:, h], x[:, 0])
    assert torch.equal(P[:, qcols + head_dim + 1], x[:, qcols + head_dim + h + 1])
    assert torch.equal(P[:, 2 * qcols:], x[:, 2 * qcols:])


@pytest.mark.parametrize("mode", [ref.GEMM_BIAS_GEGLU_SPLIT, ref.GEMM_BIAS_SWIGLU_SPLIT])
def test_gemm_reference_gated_modes_on_natural_weights(mode):
    """modes 5 and 7 on the blocked W against the natural layout: ModernBERT's gelu(in) * gate with in | gate = Wi x +
    bi (modernbert_ref._gelu), Qwen3 / Llama's silu(gate_proj x) * up_proj x (torch.nn.functional.silu)"""
    from oracle import modernbert_ref as mr
    rng = np.random.default_rng(mode)
    M, K, F = 7, 128, 192                                    # F not a multiple of 128
    ah = rng.standard_normal((M, K)).astype(np.float16)     # fp16-exact A: the lo * lo term the kernel drops is 0
    al = np.zeros_like(ah)
    A = torch.from_numpy(ah.astype(np.float64))
    w_in = (0.3 * rng.standard_normal((F, K))).astype(np.float32)
    w_gate = (0.3 * rng.standard_normal((F, K))).astype(np.float32)
    b_in = rng.standard_normal(F).astype(np.float32)
    b_gate = rng.standard_normal(F).astype(np.float32)
    wh, wl = ref.split_f16(_blocked_rows(w_in, w_gate))
    bias = _blocked_rows(b_in[:, None], b_gate[:, None])[:, 0].copy()
    out, x, S = ref.gemm_ref(mode, ah, al, wh, wl, bias)
    Win = torch.from_numpy(ref.join(*ref.split_f16(w_in)))
    Wg = torch.from_numpy(ref.join(*ref.split_f16(w_gate)))
    xin = A @ Win.T + torch.from_numpy(b_in).double()
    xg = A @ Wg.T + torch.from_numpy(b_gate).double()
    if mode == ref.GEMM_BIAS_GEGLU_SPLIT:
        want = mr._gelu(xin) * xg
    else:
        want = torch.nn.functional.silu(xin) * xg
    assert out.shape == (M, F)
    assert torch.allclose(out, want, rtol=1e-10, atol=1e-10)
    assert torch.allclose(x[:, :F], xin, rtol=1e-10, atol=1e-10) and torch.allclose(x[:, F:], xg, rtol=1e-10, atol=1e-10)
    assert torch.allclose(S[:, :F], A.abs() @ Win.abs().T, rtol=1e-12) and torch.allclose(S[:, F:], A.abs() @ Wg.abs().T,
                                                                                      rtol=1e-12)


def test_gemm_reference_fp32_residual_mode():
    rng = np.random.default_rng(6)
    M, N, K = 5, 256, 64
    a = rng.standard_normal((M, K)).astype(np.float16)
    w = rng.standard_normal((N, K)).astype(np.float16)
    z = np.zeros_like
    bias = rng.standard_normal(N).astype(np.float32)
    res = (1e5 * rng.standard_normal((M, N))).astype(np.float32)
    out, x, _ = ref.gemm_ref(ref.GEMM_BIAS_RESF32_F32, a, z(a), w, z(w), bias, res_f32=res)
    want = a.astype(np.float64) @ w.astype(np.float64).T + bias.astype(np.float64) + res.astype(np.float64)
    assert np.array_equal(out.numpy(), want)
    assert np.array_equal((out - x).numpy(), res.astype(np.float64))


def test_layernorm_reference_agrees_with_bert_ref():
    rng = np.random.default_rng(3)
    H = 384
    for offset, scale in ((0.0, 1.0), (0.0, 1e4), (3.0, 0.2)):
        x = (offset + scale * rng.standard_normal((16, H))).astype(np.float32)
        g = (1.0 + 0.1 * rng.standard_normal(H)).astype(np.float32)
        b = (0.1 * rng.standard_normal(H)).astype(np.float32)
        y, xhat, sigma = (t.numpy() for t in ref.layernorm_ref(x, g, b, 1e-12))
        want = bert_ref._layer_norm(torch.from_numpy(x), torch.from_numpy(g), torch.from_numpy(b), 1e-12).numpy()
        # bert_ref is fp32 torch: its own rounding, relative to the row's magnitude over its spread, bounds the gap
        M = np.abs(x).max(1, keepdims=True) / sigma
        assert (np.abs(y - want) <= 64 * 2.0 ** -24 * (np.abs(g) * (1 + np.abs(xhat)) * (1 + M) + np.abs(b))).all()
        assert np.allclose(xhat.mean(1), 0, atol=1e-12) and np.allclose((xhat ** 2).mean(1), 1, atol=1e-9)
    # eps inside the square root: a constant row normalises to beta, a row of variance eps to xhat / sqrt(2)
    x = np.array([[1.0, -1.0] * (H // 2)], np.float32) * np.float32(1e-6)
    y, xhat, _ = ref.layernorm_ref(x, np.ones(H, np.float32), np.zeros(H, np.float32), 1e-12)
    assert np.allclose(xhat.abs().numpy(), 1 / math.sqrt(2), rtol=1e-6)
    c = np.full((1, H), 0.375, np.float32)
    b = np.linspace(-1, 1, H, dtype=np.float32)
    assert np.array_equal(ref.layernorm_ref(c, np.ones(H, np.float32), b, 1e-12)[0].numpy()[0], b.astype(np.float64))


def _ln64(x, g, b, eps):
    mu = x.mean(1, keepdims=True)
    var = ((x - mu) ** 2).mean(1, keepdims=True)
    return (x - mu) / np.sqrt(var + np.float64(np.float32(eps))) * g.astype(np.float64) + b.astype(np.float64)


def test_embed_ln_reference_is_layernorm_of_the_three_rows():
    rng = np.random.default_rng(4)
    vocab, max_pos, type_vocab, H = 50, 6, 2, 128
    word, pos, typ = (rng.standard_normal((n, H)).astype(np.float32) for n in (vocab, max_pos, type_vocab))
    g = (1.0 + 0.1 * rng.standard_normal(H)).astype(np.float32)
    b = (0.1 * rng.standard_normal(H)).astype(np.float32)
    # an empty sequence first, in the middle and last; a sequence of exactly max_pos and one past it
    lens = [0, 3, 0, 6, 1, 8, 0]
    cu = np.r_[0, np.cumsum(lens)]
    T = int(cu[-1])
    ids = rng.integers(0, vocab, T)
    ids[0], ids[1] = -5, vocab + 7                                    # clamped to 0 and vocab - 1
    tt = rng.integers(0, 2, T)
    tt[2], tt[3] = -1, 2                                              # clamped to 0 and 1
    y, xhat, sigma, M = (t.numpy() for t in ref.embed_ln_ref(ids, tt, cu, word, pos, typ, g, b, 1e-12))
    # positions restart at every sequence and stop at max_pos - 1
    p = np.concatenate([np.minimum(np.arange(n), max_pos - 1) for n in lens])
    assert p.tolist() == [0, 1, 2, 0, 1, 2, 3, 4, 5, 0, 0, 1, 2, 3, 4, 5, 5, 5]
    ic, tc = np.clip(ids, 0, vocab - 1), np.clip(tt, 0, 1)
    x = word[ic].astype(np.float64) + typ[tc] + pos[p]
    assert np.allclose(y, _ln64(x, g, b, 1e-12), rtol=0, atol=1e-12)
    assert np.array_equal(M[:, 0], (np.abs(word[ic]).astype(np.float64) + np.abs(typ[tc]) + np.abs(pos[p])).max(1))
    assert np.allclose(sigma[:, 0], x.std(1), rtol=1e-12)
    # HF's order of the same sum in fp32 (bert_ref): within a few u of the float64 LayerNorm
    want = bert_ref._layer_norm(torch.from_numpy(word[ic] + typ[tc] + pos[p]), torch.from_numpy(g), torch.from_numpy(b),
                                1e-12).numpy()
    assert (np.abs(y - want) <= 64 * 2.0 ** -24 * (np.abs(g) * (1 + np.abs(xhat)) * (1 + M / sigma) + np.abs(b))).all()
    # no type ids = all 0
    y0 = ref.embed_ln_ref(ids, None, cu, word, pos, typ, g, b, 1e-12)[0]
    assert torch.equal(y0, ref.embed_ln_ref(ids, np.zeros(T, np.int64), cu, word, pos, typ, g, b, 1e-12)[0])


def test_pool_reference_agrees_with_bert_ref():
    rng = np.random.default_rng(5)
    H = 200
    lens = [3, 0, 1, 7, 2, 0]
    cu = np.r_[0, np.cumsum(lens)]
    T = int(cu[-1])
    hi, lo = ref.split_f16(rng.standard_normal((T, H)).astype(np.float32))
    x = ref.join(hi, lo)
    S = max(lens)
    pad = np.zeros((len(lens), S, H))
    mask = np.zeros((len(lens), S), np.int64)
    for b, n in enumerate(lens):
        pad[b, :n] = x[cu[b]:cu[b + 1]]
        mask[b, :n] = 1
    for mode, name in ((0, "mean"), (1, "cls")):
        want = bert_ref.pool(torch.from_numpy(pad), torch.from_numpy(mask), name).numpy()
        if name == "cls":
            want[np.array(lens) == 0] = 0                 # the kernel's CLS of an empty sequence is 0, not a pad row
        out, m, P = (t.numpy() for t in ref.pool_ref(hi, lo, cu, mode, False))
        assert np.allclose(out, want, rtol=1e-15, atol=1e-15) and np.array_equal(out, m)
        nrm = ref.pool_ref(hi, lo, cu, mode, True)[0].numpy()
        assert np.allclose(nrm, bert_ref.l2_normalize(torch.from_numpy(want)).numpy(), rtol=1e-14, atol=1e-15)
        assert np.allclose(np.linalg.norm(nrm[np.array(lens) > 0], axis=1), 1.0, rtol=1e-14)
        if mode == 0:
            assert np.allclose(P, np.abs(pad).sum(1), rtol=1e-15, atol=0)
        else:
            assert not P.any()
    # an empty sequence and a sequence that cancels to exactly 0 stay 0 under normalisation (no 0 / 0)
    z_hi = np.concatenate([hi[:1], -hi[:1]])
    z_lo = np.concatenate([lo[:1], -lo[:1]])
    out = ref.pool_ref(z_hi, z_lo, [0, 0, 2], 0, True)[0].numpy()
    assert np.array_equal(out, np.zeros((2, H)))
    # a 3-4-0 vector by hand
    hv, lv = ref.split_f16(np.array([[3.0, 4.0, 0.0]], np.float32))
    assert np.array_equal(ref.pool_ref(hv, lv, [0, 1], 1, True)[0].numpy(), [[0.6, 0.8, 0.0]])


def test_cls_head_reference_agrees_with_bert_ref():
    rng = np.random.default_rng(6)
    H, L = 128, 3
    lens = [2, 0, 1, 4, 0]
    cu = np.r_[0, np.cumsum(lens)]
    T = int(cu[-1])
    hi, lo = ref.split_f16(rng.standard_normal((T, H)).astype(np.float32))
    w = {"pooler.dense.weight": (rng.standard_normal((H, H)) / math.sqrt(H)).astype(np.float32),
         "pooler.dense.bias": (0.1 * rng.standard_normal(H)).astype(np.float32),
         "classifier.weight": rng.standard_normal((L, H)).astype(np.float32),
         "classifier.bias": rng.standard_normal(L).astype(np.float32)}
    args = (w["pooler.dense.weight"], w["pooler.dense.bias"], w["classifier.weight"], w["classifier.bias"])
    logits, z, pooled, A, C = (t.numpy() for t in ref.cls_head_ref(hi, lo, cu, *args))
    h = np.zeros((len(lens), H))
    for b, n in enumerate(lens):
        if n:
            h[b] = ref.join(hi, lo)[cu[b]]
    want = bert_ref.classifier_head(w, torch.from_numpy(h[:, None, :]).float()).numpy()
    assert np.allclose(logits, want, rtol=0, atol=1e-4)          # bert_ref is fp32
    W = w["pooler.dense.weight"].astype(np.float64)
    assert np.allclose(z, h @ W.T + w["pooler.dense.bias"], rtol=1e-14, atol=1e-14)
    assert np.allclose(A, np.abs(h) @ np.abs(W).T, rtol=1e-14) and np.allclose(C, np.abs(pooled) @ np.abs(args[2]).T.astype(np.float64), rtol=1e-14)
    # an empty sequence: h = 0, so the logits are W_c tanh(b_p) + b_c
    e = np.tanh(w["pooler.dense.bias"].astype(np.float64)) @ args[2].T.astype(np.float64) + args[3]
    assert np.allclose(logits[1], e, rtol=1e-14, atol=1e-14) and np.array_equal(logits[1], logits[4])
    # saturation: |z| > 20 gives tanh = +-1 exactly in float64, so the logits are signed sums of W_c rows
    pb = np.where(np.arange(H) % 2 == 0, 30.0, -30.0).astype(np.float32)
    logits, z, pooled, _, _ = (t.numpy() for t in ref.cls_head_ref(hi, lo, cu, args[0], pb, args[2], args[3]))
    assert (np.abs(z) > 20).all() and np.array_equal(np.abs(pooled), np.ones_like(pooled))
    sgn = np.sign(pb).astype(np.float64)
    assert np.allclose(logits, np.broadcast_to(args[2].astype(np.float64) @ sgn + args[3], logits.shape), rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------- the whole stack
def _ragged(ids, mask, typ):
    lens = mask.sum(1)
    cu = np.r_[0, np.cumsum(lens)]
    return (np.concatenate([ids[b, :n] for b, n in enumerate(lens)]), np.concatenate([typ[b, :n] for b, n in enumerate(lens)]),
            cu)


@pytest.mark.parametrize("preset,seed,scale", [("tiny", 0, 1.0), ("all-MiniLM-L6-v2", 1, 4.0)])
def test_stack_reference_matches_bert_ref_and_the_hf_goldens(golden_dir, preset, seed, scale):
    """float64 forward on the fp32 weights: within the oracle's own tolerances (tests/test_oracle_golden.py) of the HF
    goldens, and of bert_ref's padded fp32 forward"""
    g = np.load(f"{golden_dir}/encoder.npz")
    key = f"enc_{preset}_{seed}_{scale}"
    cfg = BertConfig(**asdict(PRESETS[preset][0]))
    w = synthetic_bert_weights(cfg, seed=seed, scale=scale)
    I, M, Ty = (g[key + s].astype(np.int64) for s in ("_ids", "_mask", "_typ"))
    ids, typ, cu = _ragged(I, M, Ty)
    out = {k: v.numpy() for k, v in ref.encoder_stack_ref(w, cfg, ids, typ, cu).items()}
    tol = 2e-5 if scale == 1.0 else 2e-4
    assert np.abs(out["mean_norm"] - g[key + "_mean"]).max() < tol
    assert np.abs(out["cls_norm"] - g[key + "_cls"]).max() < tol
    assert np.abs(out["hidden"][cu[:-1]] - g[key + "_h_first"]).max() < 50 * tol
    assert np.abs(out["hidden"][cu[1:] - 1] - g[key + "_h_last"]).max() < 50 * tol
    with torch.no_grad():
        h = bert_ref.bert_encoder_forward(w, bert_ref.BertCfg(**asdict(cfg)), *(torch.from_numpy(a) for a in (I, M, Ty)))
        mean = bert_ref.pool(h, torch.from_numpy(M), "mean")
    flat = torch.cat([h[b, :n] for b, n in enumerate(M.sum(1))]).double().numpy()
    assert np.abs(out["hidden"] - flat).max() < 1e-4
    assert np.abs(out["mean"] - mean.double().numpy()).max() < 1e-5
    assert np.abs(out["mean_norm"] - bert_ref.l2_normalize(mean).double().numpy()).max() < 1e-5


@pytest.mark.parametrize("preset,seed,scale", [("tiny", 3, 4.0), ("ms-marco-MiniLM-L-6-v2", 0, 1.0)])
def test_stack_reference_logits_match_the_hf_goldens(golden_dir, preset, seed, scale):
    g = np.load(f"{golden_dir}/cross_encoder.npz")
    key = f"ce_{preset}_{seed}_{scale}"
    cfg = BertConfig(**asdict(PRESETS[preset][0]))
    w = synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale)
    ids, typ, cu = _ragged(*(g[key + s].astype(np.int64) for s in ("_ids", "_mask", "_typ")))
    logits = ref.encoder_stack_ref(w, cfg, ids, typ, cu)["logits"].numpy()
    assert np.abs(logits - g[key + "_logits"]).max() < (2e-5 if scale == 1.0 else 5e-4)


def _small_cfg(layers, **kw):
    a = dict(vocab_size=60, hidden=128, layers=layers, heads=2, ffn=256, max_pos=16, type_vocab=2, num_labels=3)
    a.update(kw)
    return BertConfig(**a)


def test_stack_reference_layer_by_layer():
    """Layer l of the stack is the per-kernel references applied to layer l - 1's output in the encoder's order (QKV with
    q scaled by log2(e) / sqrt(d_h), attention, output projection + residual, LayerNorm, GELU FFN + residual, LayerNorm),
    and bert_ref's fp32 forward truncated to l layers agrees to fp32 accuracy.  Empty sequences first, in the middle and
    last; ids, type ids and positions out of range are clamped."""
    cfg = _small_cfg(3)
    w = synthetic_bert_weights(cfg, seed=11, with_head=True, scale=4.0)
    rng = np.random.default_rng(12)
    lens = [0, 5, 16, 0, 1, 9, 0]
    cu = np.r_[0, np.cumsum(lens)]
    T = int(cu[-1])
    ids = rng.integers(0, cfg.vocab_size, T)
    typ = rng.integers(0, 2, T)
    ids[3], ids[7], typ[4], typ[8] = -4, cfg.vocab_size + 2, -1, 5
    H, dh = cfg.hidden, cfg.hidden // cfg.heads
    V = lambda n: torch.from_numpy(w[n].astype(np.float64))  # noqa: E731
    prev = None
    for L in range(cfg.layers + 1):
        c = BertConfig(**{**asdict(cfg), "layers": L})
        got = ref.encoder_stack_ref(w, c, ids, typ, cu)
        if L == 0:
            want = ref.embed_ln_ref(ids, typ, cu, *(w["embeddings." + n] for n in (
                "word_embeddings.weight", "position_embeddings.weight", "token_type_embeddings.weight",
                "LayerNorm.weight", "LayerNorm.bias")), cfg.ln_eps)[0]
        else:
            p = f"encoder.layer.{L - 1}."
            x = prev
            q = x @ V(p + "attention.self.query.weight").T + V(p + "attention.self.query.bias")
            k = x @ V(p + "attention.self.key.weight").T + V(p + "attention.self.key.bias")
            v = x @ V(p + "attention.self.value.weight").T + V(p + "attention.self.value.bias")
            qkv = torch.cat([q * (math.log2(math.e) / math.sqrt(dh)), k, v], 1)
            ctx = ref.attention_ref(qkv, torch.zeros_like(qkv), cu, cfg.heads)[0]
            o = ctx @ V(p + "attention.output.dense.weight").T + V(p + "attention.output.dense.bias") + x
            x1 = ref.layernorm_ref(o, w[p + "attention.output.LayerNorm.weight"], w[p + "attention.output.LayerNorm.bias"],
                                   cfg.ln_eps)[0]
            f = bert_ref._gelu_erf(x1 @ V(p + "intermediate.dense.weight").T + V(p + "intermediate.dense.bias"))
            o = f @ V(p + "output.dense.weight").T + V(p + "output.dense.bias") + x1
            want = ref.layernorm_ref(o, w[p + "output.LayerNorm.weight"], w[p + "output.LayerNorm.bias"], cfg.ln_eps)[0]
        assert torch.allclose(got["hidden"], want, rtol=0, atol=1e-12), f"layer {L}"
        prev = got["hidden"]
        # bert_ref in fp32, padded, on the clamped inputs (it indexes the tables directly)
        S = max(lens)
        I = np.zeros((len(lens), S), np.int64); M = np.zeros_like(I); Ty = np.zeros_like(I)
        for b, n in enumerate(lens):
            I[b, :n] = np.clip(ids[cu[b]:cu[b + 1]], 0, cfg.vocab_size - 1)
            Ty[b, :n] = np.clip(typ[cu[b]:cu[b + 1]], 0, 1)
            M[b, :n] = 1
        with torch.no_grad():
            h = bert_ref.bert_encoder_forward(w, bert_ref.BertCfg(**asdict(c)), *(torch.from_numpy(a) for a in (I, M, Ty)))
        flat = torch.cat([h[b, :n] for b, n in enumerate(lens)]).double()
        assert (got["hidden"] - flat).abs().max() < 2e-5, f"layer {L} vs bert_ref"
    # the outputs of the last layer: pooling and head rules, empty sequences included
    empty = np.diff(cu) == 0
    for name in ("mean", "cls", "mean_norm", "cls_norm"):
        assert (got[name][torch.from_numpy(empty)] == 0).all()
    e = np.tanh(w["pooler.dense.bias"].astype(np.float64)) @ w["classifier.weight"].T.astype(np.float64) + w["classifier.bias"]
    assert np.allclose(got["logits"].numpy()[empty], e, rtol=0, atol=1e-14)
    assert torch.equal(got["cls"][torch.from_numpy(~empty)], got["hidden"][torch.from_numpy(cu[:-1][~empty])])


def test_stack_reference_on_split_weights_is_the_forward_on_hi_plus_lo():
    """weights="split" is exactly the fp32 forward on fp32(hi + lo) (hi + lo has at most 22 significant bits, so it is
    an fp32 value), and only the GEMM weights are split"""
    cfg = _small_cfg(2)
    w = synthetic_bert_weights(cfg, seed=13, with_head=True, scale=1.0)
    ws = dict(w)
    for name in w:
        if name.endswith(ref.GEMM_WEIGHTS):
            hi, lo = ref.split_f16(w[name])
            joined = ref.join(hi, lo)
            assert np.array_equal(joined.astype(np.float32).astype(np.float64), joined)
            ws[name] = joined.astype(np.float32)
            assert np.array_equal(ref.split_weight(w[name]).numpy(), joined)
    assert sum(n.endswith(ref.GEMM_WEIGHTS) for n in w) == 6 * cfg.layers
    rng = np.random.default_rng(14)
    # a subnormal lo plane: |w| ~ 0.02 keeps its error under max(2^-22 |w|, 2^-25); most weights exceed 2^-22 |w|
    x = (0.02 * rng.standard_normal(100000)).astype(np.float32)
    err = np.abs(ref.split_weight(x).numpy() - x.astype(np.float64))
    assert (err <= np.maximum(2.0 ** -22 * np.abs(x), 2.0 ** -25)).all()
    assert (err > 2.0 ** -22 * np.abs(x)).mean() > 0.5
    lens = [3, 0, 16, 7]
    cu = np.r_[0, np.cumsum(lens)]
    ids = rng.integers(0, cfg.vocab_size, cu[-1])
    a = ref.encoder_stack_ref(w, cfg, ids, None, cu, weights="split")
    b = ref.encoder_stack_ref(ws, cfg, ids, None, cu, weights="fp32")
    for k in a:
        assert torch.equal(a[k], b[k]), k


# What the split weights cost, measured (float64 forward on hi + lo against the float64 forward on the fp32 weights,
# synthetic weights, 4 sequences of 96 tokens), beside what a plain fp32 forward (bert_ref) costs against the same
# float64 result: (hidden max, hidden rms, normalised mean-embedding max) for each.  Pinned within a factor of 1.5 either
# way: the representation costs up to ~1.7x fp32's hidden-state error and ~7x its error on normalised embeddings.
REP_COST = {
    ("all-MiniLM-L6-v2", 1.0): ((2.95e-6, 5.89e-7, 1.19e-7), (3.59e-6, 3.14e-7, 6.09e-8)),
    ("all-MiniLM-L6-v2", 4.0): ((3.31e-6, 9.14e-7, 1.67e-7), (3.66e-6, 6.81e-7, 6.80e-8)),
    ("bge-base-en-v1.5", 1.0): ((8.80e-6, 1.67e-6, 2.16e-7), (5.10e-6, 6.41e-7, 3.09e-8)),
}


@pytest.mark.parametrize("preset,scale", list(REP_COST))
def test_split_weight_representation_cost(preset, scale):
    cfg = BertConfig(**asdict(PRESETS[preset][0]))
    w = synthetic_bert_weights(cfg, seed=3, scale=scale)
    rng = np.random.default_rng(5)
    lens = [96] * 4
    ids = rng.integers(104, cfg.vocab_size, sum(lens))
    cu = np.r_[0, np.cumsum(lens)]
    a = ref.encoder_stack_ref(w, cfg, ids, None, cu, "fp32")
    b = ref.encoder_stack_ref(w, cfg, ids, None, cu, "split")
    I = torch.from_numpy(ids.reshape(4, 96))
    with torch.no_grad():
        h = bert_ref.bert_encoder_forward(w, bert_ref.BertCfg(**asdict(cfg)), I, torch.ones_like(I))
        e32 = bert_ref.l2_normalize(h.mean(1)).double()
    h32 = h.reshape(-1, cfg.hidden).double()

    def costs(h_, e_):
        d = (h_ - a["hidden"]).abs()
        return float(d.max()), float(d.pow(2).mean().sqrt()), float((e_ - a["mean_norm"]).abs().max())

    for what, got, want in (("split", costs(b["hidden"], b["mean_norm"]), REP_COST[preset, scale][0]),
                            ("fp32", costs(h32, e32), REP_COST[preset, scale][1])):
        for g_, w_, name in zip(got, want, ("hidden max", "hidden rms", "embedding max")):
            assert w_ / 1.5 <= g_ <= 1.5 * w_, f"{what} {name}: {g_:.3g}, pinned {w_:.3g}"
