"""CPU: the float64 per-kernel references (oracle/encoder_kernels_ref.py) against independent restatements, so that
tests/test_encoder_kernels_gpu.py judges the kernels against something that is itself pinned."""
import math

import numpy as np
import torch

from oracle import bert_ref
from oracle import encoder_kernels_ref as ref


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
