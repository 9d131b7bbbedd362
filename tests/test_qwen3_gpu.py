"""Qwen3 on the GPU encoder: each new kernel against float64 through its debug entry (RMSNorm to split planes, the q / k
norm + rotary step, causal grouped-query attention at head_dim 128, the SwiGLU epilogue, the last-token rows), then the
whole stack against the float64 forward, the goldens and the fp32 oracle, and the product classes end to end."""
from __future__ import annotations

import gc
import importlib.util
import math
import os
from dataclasses import asdict, replace

import numpy as np
import pytest
import torch

from oracle import encoder_kernels_ref as ref
from oracle import qwen3_ref as qr
from ragmeup_b200.documents import Document
from ragmeup_b200.weights import PRESETS, Qwen3Config, rope_table, synthetic_qwen3_weights

pytestmark = pytest.mark.gpu
LOG2E = math.log2(math.e)
# the whole stack's max and RMS error against float64 may be at most this multiple of the fp32 forward's (fixed before
# the first run; the measured ratios are in DESIGN.md)
STACK_RATIO = 32.0


def _lib():
    from ragmeup_b200 import _lib
    return _lib


@pytest.fixture(autouse=True)
def _release_torch_cache():
    """the encoder allocates with cudaMalloc, outside torch's caching allocator: hand back what earlier tests' float64
    references left cached, and keep fp32 matmuls out of TF32"""
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _ptr(t):
    return None if t is None else t.data_ptr()


def _planes(x):
    return [torch.from_numpy(p).cuda() for p in ref.split_f16(np.ascontiguousarray(x, dtype=np.float32))]


def _j(p):
    return p[0].double() + p[1].double()


def _golden_module():
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden_qwen3.py")
    spec = importlib.util.spec_from_file_location("make_golden_qwen3", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _tiny(**kw):
    return replace(Qwen3Config(**asdict(PRESETS["tiny-qwen3"][0])), **kw)


# ------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("H", [128, 1024, 2560, 4096])
@pytest.mark.parametrize("T", [1, 7, 4097])
def test_rmsnorm_split_matches_float64(cuda, H, T):
    L = _lib()
    rng = np.random.default_rng(H + T)
    x = (rng.standard_normal((T, H)) * rng.uniform(0.1, 30.0, (T, 1))).astype(np.float32)
    w = (1.0 + 0.2 * rng.standard_normal(H)).astype(np.float32)
    xd, wd = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda()
    hi = torch.full((T, H), float("nan"), dtype=torch.float16, device="cuda")
    lo = torch.full_like(hi, float("nan"))
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(L.lib().rmu_debug_rmsnorm(_ptr(xd), T, H, _ptr(wd), 1e-6, _ptr(hi), _ptr(lo), _ptr(flag), L.stream_ptr()), "rmsnorm")
    torch.cuda.synchronize()
    X = xd.double()
    want = wd.double() * (X * torch.rsqrt(X.pow(2).mean(-1, keepdim=True) + 1e-6))
    got = hi.double() + lo.double()
    err = float(((got - want).abs() / want.abs().amax(1, keepdim=True)).max())
    print(f"\nrmsnorm H={H} T={T}: max |err| / row max = {err:.3g}")
    assert err <= 2e-6 and int(flag.item()) == 0
    # a row past the fp16 range sets the flag
    w_big = torch.full_like(wd, 1e5)
    L.check(L.lib().rmu_debug_rmsnorm(_ptr(xd), 1, H, _ptr(w_big), 1e-6, _ptr(hi), _ptr(lo), _ptr(flag), L.stream_ptr()), "rmsnorm")
    torch.cuda.synchronize()
    assert int(flag.item()) == 1


@pytest.mark.parametrize("heads,kv", [(16, 8), (4, 4), (8, 2)])
def test_qk_norm_rope_matches_float64(cuda, heads, kv):
    """per-head RMSNorm of q and k, rotate-half rotary at positions up to 8191, q times log2(e) / sqrt(128), v as it is"""
    L = _lib()
    rng = np.random.default_rng(heads * 10 + kv)
    T, d, NH = 700, 128, heads + 2 * kv
    x = (rng.standard_normal((T, NH * d)) * 3.0).astype(np.float32)
    pos = rng.integers(0, 8192, T).astype(np.int32)
    pos[:4] = [0, 1, 8190, 8191]
    qn = (1.0 + 0.2 * rng.standard_normal(d)).astype(np.float32)
    kn = (1.0 + 0.2 * rng.standard_normal(d)).astype(np.float32)
    cos, sin = rope_table(1000000.0, d, 8192)
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in
           dict(x=x, pos=pos, qn=qn, kn=kn, cos=cos, sin=sin).items()}
    hi = torch.full((T, NH * d), float("nan"), dtype=torch.float16, device="cuda")
    lo = torch.full_like(hi, float("nan"))
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    qs = LOG2E / math.sqrt(d)
    L.check(L.lib().rmu_debug_qk_norm_rope(_ptr(dev["x"]), T, heads, kv, _ptr(dev["pos"]), _ptr(dev["qn"]), _ptr(dev["kn"]),
                                           1e-6, qs, _ptr(dev["cos"]), _ptr(dev["sin"]), 8192, _ptr(hi), _ptr(lo),
                                           _ptr(flag), L.stream_ptr()), "qk_norm_rope")
    torch.cuda.synchronize()
    X = dev["x"].double().view(T, NH, d)
    c = dev["cos"].double()[dev["pos"].long()][:, None, :]
    s = dev["sin"].double()[dev["pos"].long()][:, None, :]
    c, s = torch.cat([c, c], -1), torch.cat([s, s], -1)

    def norm_rope(v, w):
        y = w * (v * torch.rsqrt(v.pow(2).mean(-1, keepdim=True) + 1e-6))
        return y * c + torch.cat([-y[..., d // 2:], y[..., :d // 2]], -1) * s
    want = X.clone()
    want[:, :heads] = norm_rope(X[:, :heads], dev["qn"].double()) * qs
    want[:, heads:heads + kv] = norm_rope(X[:, heads:heads + kv], dev["kn"].double())
    got = (hi.double() + lo.double()).view(T, NH, d)
    err = float(((got - want).abs() / want.abs().amax(-1, keepdim=True)).max())
    print(f"\nqk_norm_rope heads={heads} kv={kv}: max |err| / head max = {err:.3g}")
    assert err <= 2e-6 and int(flag.item()) == 0
    assert torch.equal(got[:, heads + kv:], (_j(_planes(x)).view(T, NH, d))[:, heads + kv:])


def _attention(qkv, cu, heads, kv, max_len):
    L = _lib()
    T = int(cu[-1])
    ph, pl = _planes(qkv)
    cu_d = torch.from_numpy(np.asarray(cu, np.int32)).cuda()
    oh = torch.full((T, heads * 128), float("nan"), dtype=torch.float16, device="cuda")
    ol = torch.full_like(oh, float("nan"))
    L.check(L.lib().rmu_debug_attention_causal(_ptr(ph), _ptr(pl), _ptr(cu_d), len(cu) - 1, heads, kv, int(max_len),
                                               _ptr(oh), _ptr(ol), L.stream_ptr()), "attention_causal")
    torch.cuda.synchronize()
    return (ph, pl), oh.double() + ol.double()


def _attention_ref(planes, cu, heads, kv):
    """float64 causal GQA on the split operands: p_ij proportional to 2^(q'_i . k_j) for j <= i (q' pre-scaled)"""
    d, G = 128, heads // kv
    X = _j(planes)
    out = torch.zeros(X.shape[0], heads * d, dtype=torch.float64, device="cuda")
    for b in range(len(cu) - 1):
        t0, t1 = int(cu[b]), int(cu[b + 1])
        S = t1 - t0
        if S == 0:
            continue
        mask = torch.ones(S, S, dtype=torch.bool, device="cuda").tril()
        for h in range(heads):
            q = X[t0:t1, h * d:(h + 1) * d]
            k = X[t0:t1, (heads + h // G) * d:(heads + h // G + 1) * d]
            v = X[t0:t1, (heads + kv + h // G) * d:(heads + kv + h // G + 1) * d]
            s = (q @ k.T * math.log(2.0)).masked_fill(~mask, float("-inf")).softmax(-1)
            out[t0:t1, h * d:(h + 1) * d] = s @ v
    return out


ATT_CASES = [([1], 2, 2), ([15, 16, 17], 4, 2), ([127, 128, 129], 4, 1), ([1000], 4, 4), ([8192], 2, 1),
             ([1, 15, 16, 17, 127, 128, 129, 1000, 3], 8, 2), ([129, 0, 1000, 17, 1], 4, 1), ([300, 45], 8, 8)]


@pytest.mark.parametrize("lens,heads,kv", ATT_CASES)
def test_causal_attention_matches_float64(cuda, lens, heads, kv):
    """lengths around the 16 / 32 / 64 / 128-row blocks, up to 8192, ragged and with an empty sequence; group sizes
    heads / kv of 1, 2 and 4"""
    rng = np.random.default_rng(sum(lens) + heads)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    T, NH = int(cu[-1]), heads + 2 * kv
    qkv = rng.standard_normal((T, NH * 128)).astype(np.float32)
    qkv[:, :heads * 128] *= 0.3                       # scores of a few units in log2: peaked but not one-hot
    planes, got = _attention(qkv, cu, heads, kv, max(lens))
    want = _attention_ref(planes, cu, heads, kv)
    vmax = float(_j(planes)[:, (heads + kv) * 128:].abs().max())
    err = float((got - want).abs().max())
    print(f"\nattention {lens} heads={heads} kv={kv}: max |err| / max|v| = {err / vmax:.3g}")
    assert torch.isfinite(got).all() and err <= 2e-5 * vmax


def test_causal_attention_equal_scores(cuda):
    """q = 0: every visible key weighs the same, so row i is the running mean of v over j <= i"""
    heads, kv, lens = 4, 2, [1, 33, 700]
    rng = np.random.default_rng(5)
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    qkv = rng.standard_normal((int(cu[-1]), (heads + 2 * kv) * 128)).astype(np.float32)
    qkv[:, :heads * 128] = 0.0
    planes, got = _attention(qkv, cu, heads, kv, max(lens))
    want = _attention_ref(planes, cu, heads, kv)
    X = _j(planes)
    t0, t1 = int(cu[2]), int(cu[3])
    v0 = X[t0:t1, (heads + kv) * 128:(heads + kv + 1) * 128]
    mean = v0.cumsum(0) / torch.arange(1, t1 - t0 + 1, device="cuda", dtype=torch.float64)[:, None]
    assert float((want[t0:t1, :128] - mean).abs().max()) < 1e-12
    assert float((got - want).abs().max()) <= 2e-5 * float(X.abs().max())


def test_causal_attention_70000_one_token_sequences(cuda):
    """more than 65 535 sequences run in grid-y slices; a one-token sequence's context is its own v"""
    heads, kv, B = 4, 2, 70000
    rng = np.random.default_rng(6)
    cu = np.arange(B + 1, dtype=np.int32)
    qkv = rng.standard_normal((B, (heads + 2 * kv) * 128)).astype(np.float32)
    planes, got = _attention(qkv, cu, heads, kv, 1)
    X = _j(planes)
    want = torch.cat([X[:, (heads + kv + h // 2) * 128:(heads + kv + h // 2 + 1) * 128] for h in range(heads)], 1)
    assert float((got - want).abs().max()) <= 1e-6 * float(X.abs().max())


def _swiglu_rows(gate, up):
    """rmu_encoder_create_qwen3's reorder of gate | up: 128-row blocks of 64 gate rows, then the 64 matching up rows"""
    F = gate.shape[0]
    out = np.empty((2 * F, gate.shape[1]), np.float32)
    for k in range(F // 64):
        out[128 * k:128 * k + 64] = gate[64 * k:64 * k + 64]
        out[128 * k + 64:128 * k + 128] = up[64 * k:64 * k + 64]
    return out


def _swiglu(a, wp, M, N, K, flag):
    L = _lib()
    bias = torch.zeros(N, dtype=torch.float32, device="cuda")
    oh = torch.full((M, N // 2), float("nan"), dtype=torch.float16, device="cuda")
    ol = torch.full_like(oh, float("nan"))
    L.check(L.lib().rmu_debug_gemm_swiglu(_ptr(a[0]), _ptr(a[1]), a[0].shape[0], _ptr(wp[0]), _ptr(wp[1]), M, N, K, _ptr(bias), 0,
                                          _ptr(oh), _ptr(ol), _ptr(flag), L.stream_ptr()), "gemm_swiglu")
    torch.cuda.synchronize()
    return oh.double() + ol.double()


@pytest.mark.parametrize("F", [384, 3072])
def test_swiglu_epilogue_matches_float64(cuda, F):
    """silu(gate) * up against float64 on the split operands, F = 3072 the 0.6B shape; a tile past fp16's range sets
    the flag, and NaN rows of A past M (read by the last row tile, clipped from the output) do not"""
    rng = np.random.default_rng(F)
    M, K = 300, 256
    a_full = rng.standard_normal((M + 60, K)).astype(np.float32)
    a_full[M:] = np.nan
    a = _planes(a_full)
    gate = (rng.standard_normal((F, K)) * 0.1).astype(np.float32)
    up = (rng.standard_normal((F, K)) * 0.1).astype(np.float32)
    wp = _planes(_swiglu_rows(gate, up))
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    got = _swiglu(a, wp, M, 2 * F, K, flag)
    A = _j(a)[:M]
    G, U = A @ _j(_planes(gate)).T, A @ _j(_planes(up)).T
    Ga, Ua = A.abs() @ _j(_planes(gate)).abs().T, A.abs() @ _j(_planes(up)).abs().T
    want = torch.nn.functional.silu(G) * U
    bound = 2.0 ** -19 * (Ga * U.abs() + torch.nn.functional.silu(G).abs() * Ua) + 2.0 ** -21 * want.abs() + 1e-30
    ratio = float(((got - want).abs() / bound).max())
    print(f"\nswiglu F={F}: max |err| / bound = {ratio:.3g}")
    assert ratio <= 1.0 and int(flag.item()) == 0
    big = _planes(_swiglu_rows(gate * 1000.0, up * 1000.0))
    _swiglu(a, big, M, 2 * F, K, flag)
    assert int(flag.item()) == 1


@pytest.mark.parametrize("mode", ["normalize", "plain", "head"])
def test_last_token_rows_match_float64(cuda, mode):
    """the row rule (last token, or the rightmost id != pad_id; the first when all are pads; zeros when empty), RMSNorm,
    then L2-normalise or the [num_labels, H] head"""
    L = _lib()
    rng = np.random.default_rng(7)
    H, lens = 2560, [5, 1, 0, 9, 4, 300]
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    T, B = int(cu[-1]), len(lens)
    pad = 7 if mode == "head" else -1
    ids = rng.integers(10, 100, T).astype(np.int32)
    ids[cu[1] - 2:cu[1]] = 7                                  # ends with two pads
    ids[cu[4]:cu[5]] = 7                                      # all pads
    ids[cu[6] - 40:cu[6]] = 7                                 # a pad run across a 32-token window
    x = (rng.standard_normal((T, H)) * 5).astype(np.float32)
    w = (1.0 + 0.2 * rng.standard_normal(H)).astype(np.float32)
    nl = 3
    head = (rng.standard_normal((nl, H)) * 0.05).astype(np.float32)
    d = {k: torch.from_numpy(v).cuda() for k, v in dict(x=x, ids=ids, cu=cu, w=w, head=head).items()}
    out = torch.full((B, nl if mode == "head" else H), float("nan"), dtype=torch.float32, device="cuda")
    L.check(L.lib().rmu_debug_last_token(_ptr(d["x"]), _ptr(d["ids"]), _ptr(d["cu"]), B, H, _ptr(d["w"]), 1e-6, pad,
                                         int(mode == "normalize"), _ptr(d["head"]) if mode == "head" else None, nl,
                                         _ptr(out), L.stream_ptr()), "last_token")
    torch.cuda.synchronize()
    X = d["x"].double()
    want = torch.zeros_like(out, dtype=torch.float64)
    for b in range(B):
        if lens[b] == 0:
            continue
        r = cu[b] + qr.head_row(ids[cu[b]:cu[b + 1]].tolist(), pad)
        y = d["w"].double() * (X[r] * torch.rsqrt(X[r].pow(2).mean() + 1e-6))
        if mode == "normalize":
            y = y / y.norm()
        want[b] = d["head"].double() @ y if mode == "head" else y
    err = float((out.double() - want).abs().max() / want.abs().max())
    print(f"\nlast token {mode}: max |err| / max = {err:.3g}")
    assert err <= 2e-6 and torch.equal(out[2], torch.zeros_like(out[2]))


# ------------------------------------------------------------------------------------------------- the stack
def _encoder(cfg, w, with_head):
    from ragmeup_b200.encoder import BertEncoder
    return BertEncoder(cfg, w, with_head=with_head, device=0)


def _batch(cfg, lens, seed):
    rng = np.random.default_rng(seed)
    seqs = [rng.integers(0, cfg.vocab_size, n).tolist() for n in lens]
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    return seqs, np.concatenate([np.asarray(s, np.int32) for s in seqs]), cu


def _stack_errors(cfg, w, lens, seed):
    """(gpu, fp32) max and RMS error of every hidden row against float64"""
    enc = _encoder(cfg, w, False)
    seqs, ids, cu = _batch(cfg, lens, seed)
    got = enc.hidden_tokens(ids, None, cu, max(lens)).double()
    W64, W32 = qr.weights(w, torch.float64, "cuda"), qr.weights(w, torch.float32, "cuda")
    want = torch.cat([qr.hidden(W64, cfg, s, torch.float64) for s in seqs])
    f32 = torch.cat([qr.hidden(W32, cfg, s, torch.float32) for s in seqs]).double()
    e_gpu, e_32 = (got - want).abs(), (f32 - want).abs()
    return (float(e_gpu.max()), float(e_gpu.pow(2).mean().sqrt())), (float(e_32.max()), float(e_32.pow(2).mean().sqrt()))


@pytest.mark.parametrize("shape", ["tiny-qwen3", "qwen3-embedding-0.6b"])
def test_qwen3_stack_matches_float64_forward(cuda, shape):
    cfg = Qwen3Config(**asdict(PRESETS[shape][0]))
    w = synthetic_qwen3_weights(cfg, seed=11, scale=2.0)
    lens = [1, 17, 129, 600] if shape == "tiny-qwen3" else [1, 40, 300]
    (gm, gr), (fm, fr) = _stack_errors(cfg, w, lens, 12)
    print(f"\n{shape}: gpu max {gm:.3g} rms {gr:.3g}; fp32 max {fm:.3g} rms {fr:.3g}; ratios {gm / fm:.3g} {gr / fr:.3g}")
    assert gm <= STACK_RATIO * fm and gr <= STACK_RATIO * fr


def test_goldens(cuda, golden_dir):
    """embeddings, sequence-classification logits and reranker scores of transformers' fp32 models, from the stored ids"""
    g = np.load(os.path.join(golden_dir, "qwen3.npz"))
    mod = _golden_module()
    cfg, w, lm, _tok = mod.build()
    body = {k: v for k, v in w.items() if k != "head"}
    emb = _encoder(cfg, body, False).embed_tokens(g["emb_ids"], None, g["emb_cu"], int(np.diff(g["emb_cu"]).max()),
                                                  "last", True).cpu().numpy()
    assert np.abs(emb - g["emb"]).max() < 1e-3
    cls = _encoder(cfg, w, True).classify_tokens(g["cls_ids"], None, g["cls_cu"], int(np.diff(g["cls_cu"]).max())).cpu().numpy()
    assert np.abs(cls - g["cls_logits"]).max() < 1e-3
    yes, no = (int(i) for i in g["yes_no"])
    rcfg = replace(cfg, reranker=True, num_labels=2)
    rr = _encoder(rcfg, {**body, "head": lm[[no, yes]]}, True).classify_tokens(g["rr_ids"], None, g["rr_cu"],
                                                                              int(np.diff(g["rr_cu"]).max()))
    from ragmeup_b200.cross_encoder import yes_probability
    assert np.abs(yes_probability(rr.cpu().numpy()) - g["rr_scores"]).max() < 1e-3


def test_embeddings_and_scores_match_fp32_oracle(cuda):
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    mod = _golden_module()
    emb = HuggingFaceEmbeddings(model_name="synthetic:tiny-qwen3:4:2.0")
    texts = mod.texts(20, 1, 300, 21)
    got = np.asarray(emb.embed_documents(texts), np.float32)
    ids, _t, cu = emb._ragged(texts)
    W = qr.weights(synthetic_qwen3_weights(emb.config, 4, False, 2.0), torch.float32, "cuda")
    want = qr.embed(W, emb.config, [ids[cu[b]:cu[b + 1]].tolist() for b in range(len(texts))], True, torch.float32)
    assert np.abs(got - want.cpu().numpy()).max() < 1e-3
    ce = HuggingFaceCrossEncoder(model_name="synthetic:tiny-qwen3:5:2.0")
    pairs = [(q, d) for q in mod.texts(3, 2, 8, 22) for d in mod.texts(6, 10, 200, 23)]
    s = ce.score(pairs)
    ids, _t, cu = ce._pairs([p[0] for p in pairs], [p[1] for p in pairs])
    W = qr.weights(synthetic_qwen3_weights(ce.config, 5, True, 2.0), torch.float32, "cuda")
    lg = qr.logits(W, ce.config, [ids[cu[b]:cu[b + 1]].tolist() for b in range(len(pairs))], ce.config.head_pad_id,
                   torch.float32)
    assert np.abs(s - torch.sigmoid(lg[:, 0]).cpu().numpy()).max() < 1e-3
    assert np.abs(ce.score_tensor(pairs).cpu().numpy() - s).max() < 1e-6


@pytest.fixture(scope="module")
def snapshots(tmp_path_factory):
    pytest.importorskip("transformers")
    mod = _golden_module()
    cfg, w, lm, tok = mod.build()
    root = tmp_path_factory.mktemp("qwen3")
    return mod, cfg, w, lm, tok, mod.save_snapshots(str(root), cfg, w, lm, tok)


def test_snapshots_end_to_end(cuda, snapshots):
    """saved Qwen3Model / Qwen3ForSequenceClassification / Qwen3ForCausalLM snapshots through HuggingFaceEmbeddings, a
    Milvus store with MMR and both cross-encoder forms, against transformers on the same ids"""
    import transformers
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.reranker import ScoredCrossEncoderReranker
    from ragmeup_b200.vectorstore import Milvus
    mod, cfg, w, lm, tok, dirs = snapshots
    emb = HuggingFaceEmbeddings(model_name=dirs["embedder"])
    assert emb.pooling == "last" and emb.normalize and emb.max_seq_length == 1024
    docs = mod.texts(60, 10, 80, 30)
    got = np.asarray(emb.embed_documents(docs[:8]), np.float32)
    base = transformers.Qwen3Model.from_pretrained(dirs["embedder"], attn_implementation="eager").eval()
    with torch.no_grad():
        want = np.stack([torch.nn.functional.normalize(base(torch.tensor([tok.encode(t).ids])).last_hidden_state[0, -1],
                                                       dim=-1).numpy() for t in docs[:8]])
    assert np.abs(got - want).max() < 1e-3
    db = Milvus.from_documents([], emb, drop_old=True, connection_args={"uri": "data.db"}, collection_name="qwen3")
    db.add_documents([Document(t, {"id": f"id{i}"}) for i, t in enumerate(docs)], ids=[f"id{i}" for i in range(60)])
    retriever = db.as_retriever(search_type="mmr", search_kwargs={"k": 10})
    seqcls = HuggingFaceCrossEncoder(model_name=dirs["seqcls"])
    rer = HuggingFaceCrossEncoder(model_name=dirs["reranker"])
    assert seqcls.activation == "sigmoid" and rer.activation == "yes_prob" and rer.config.reranker
    seq_m = transformers.Qwen3ForSequenceClassification.from_pretrained(dirs["seqcls"], attn_implementation="eager").eval()
    lm_m = transformers.Qwen3ForCausalLM.from_pretrained(dirs["reranker"], attn_implementation="eager").eval()
    yes, no = tok.token_to_id("yes"), tok.token_to_id("no")
    for qtext in mod.texts(2, 3, 8, 31):
        found = retriever.invoke(qtext)
        assert len(found) == 10
        pairs = [(qtext, d.page_content) for d in found]
        for ce in (seqcls, rer):
            s = ce.score(pairs)
            ids, _t, cu = ce._pairs([p[0] for p in pairs], [p[1] for p in pairs])
            with torch.no_grad():
                if ce is seqcls:
                    ref_s = [float(torch.sigmoid(seq_m(torch.tensor([ids[cu[b]:cu[b + 1]].tolist()])).logits[0, 0]))
                             for b in range(len(pairs))]
                else:
                    ref_s = []
                    for b in range(len(pairs)):
                        lg = lm_m(torch.tensor([ids[cu[b]:cu[b + 1]].tolist()])).logits[0, -1]
                        ref_s.append(float(torch.stack([lg[no], lg[yes]]).log_softmax(0)[1].exp()))
            assert np.abs(s - np.asarray(ref_s, np.float32)).max() < 1e-3
            top = ScoredCrossEncoderReranker(model=ce, top_n=3).compress_documents(found, qtext)
            order = sorted(range(len(found)), key=lambda i: s[i], reverse=True)[:3]
            assert [d.page_content for d in top] == [found[i].page_content for i in order]


def test_bf16_snapshot_scores_as_its_fp32_weights(cuda, snapshots, tmp_path):
    """a bfloat16 save loads widened to float32 and scores as the encoder does on those widened weights"""
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    mod, cfg, w, lm, tok, _dirs = snapshots
    dirs = mod.save_snapshots(str(tmp_path), cfg, w, lm, tok, bf16=True)
    ce = HuggingFaceCrossEncoder(model_name=dirs["seqcls"])
    pairs = [(q, d) for q in mod.texts(2, 2, 6, 40) for d in mod.texts(3, 10, 60, 41)]
    s = ce.score(pairs)
    ids, _t, cu = ce._pairs([p[0] for p in pairs], [p[1] for p in pairs])
    wb = {k: torch.from_numpy(v).to(torch.bfloat16).float().numpy() for k, v in w.items()}
    lg = qr.logits(qr.weights(wb, torch.float32, "cuda"), ce.config, [ids[cu[b]:cu[b + 1]].tolist() for b in range(len(pairs))],
                   ce.config.head_pad_id, torch.float32)
    assert np.abs(s - torch.sigmoid(lg[:, 0]).cpu().numpy()).max() < 1e-3


def test_sequence_past_max_pos_is_refused(cuda):
    from ragmeup_b200._lib import RmuError
    cfg = _tiny(max_pos=256)
    enc = _encoder(cfg, synthetic_qwen3_weights(cfg, 0), False)
    ids = np.ones(257, np.int32)
    with pytest.raises(RmuError, match="max_position_embeddings"):
        enc.embed_tokens(ids, None, np.asarray([0, 257], np.int32), 257, "last", True)
    assert enc.embed_tokens(ids[:256], None, np.asarray([0, 256], np.int32), 256, "last", True).shape == (1, cfg.hidden)


def test_fp16_range_guard_raises_naming_the_model(cuda):
    """gate / up weights scaled so the SwiGLU output passes 65504: the forward raises instead of returning inf / NaN"""
    from ragmeup_b200._lib import RmuError
    cfg = _tiny(name="synthetic:tiny-qwen3-overflow")
    w = synthetic_qwen3_weights(cfg, 0)
    for l in range(cfg.layers):
        for k in ("mlp.gate_proj.weight", "mlp.up_proj.weight"):
            w[f"layers.{l}.{k}"] = w[f"layers.{l}.{k}"] * 1000.0
    enc = _encoder(cfg, w, False)
    seqs, ids, cu = _batch(cfg, [5, 40], 3)
    with pytest.raises(RmuError, match="synthetic:tiny-qwen3-overflow.*fp16 range"):
        enc.embed_host(ids, None, cu, "last", True)
    with pytest.raises(RmuError, match="fp16 range"):
        enc.hidden_tokens(ids, None, cu, 40)


def test_last_token_pooling_is_qwen3_only(cuda):
    """a BERT encoder still refuses RMU_POOL_LAST, and a Qwen3 encoder refuses mean and CLS pooling"""
    from ragmeup_b200._lib import RmuError
    from ragmeup_b200.weights import BertConfig, synthetic_bert_weights
    bcfg = BertConfig(**asdict(PRESETS["all-MiniLM-L6-v2"][0]))
    benc = _encoder(bcfg, synthetic_bert_weights(bcfg, 0), False)
    ids, cu = np.full(5, 1000, np.int32), np.asarray([0, 5], np.int32)
    with pytest.raises(RmuError, match="pool_mode"):
        benc.embed_tokens(ids, None, cu, 5, "last", True)
    cfg = _tiny()
    qenc = _encoder(cfg, synthetic_qwen3_weights(cfg, 0), False)
    for pooling in ("mean", "cls"):
        with pytest.raises(RmuError, match="last token"):
            qenc.embed_tokens(ids, None, cu, 5, pooling, True)
