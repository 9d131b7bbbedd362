"""GPU: the whole encoder (rmu_encoder_hidden, _embed, _classify and the _host variants) against the float64 forward of
oracle/encoder_kernels_ref.py on the SPLIT weights (hi + lo, as rmu_encoder_create uploads them), so that what is left
is the kernels' arithmetic alone, across the model shapes rmu_encoder_create accepts; then the batch and call limits:
more than 65 535 sequences, the Python chunking at MAX_TOKENS_PER_CALL, workspace growth and max_seqlen.

The bar is relative to what fp32 achieves.  err_32 is the error of a plain fp32 forward (oracle.bert_ref, torch on the
device with TF32 off, on the same split weights) against the same float64 result.  The GPU's max and RMS errors must
each be within c x err_32 plus a floor of FLOOR u |output| (max or RMS of the output), which keeps an exactly computed
output from having a zero bound; c is set per case from the measured ratios, which are in DESIGN.md section 2 and
printed here (-s).  The encoder's error is 5 to 30 times fp32's: E1 adds each k16 step with rounding toward zero, so its
accumulation error grows as sqrt(K) without cancelling (tests/test_encoder_kernels_gpu.py), and it compounds with depth.
"""
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import bert_ref
from oracle import encoder_kernels_ref as ref
from ragmeup_b200.weights import PRESETS, BertConfig, synthetic_bert_weights

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
FLOOR = 4.0
OUTPUTS = ("hidden", "mean", "mean_norm", "cls", "cls_norm", "logits")


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _preset(name, **kw):
    return BertConfig(**{**asdict(PRESETS[name][0]), **kw})


def _cfg(H, heads, F, layers, labels, **kw):
    return BertConfig(**{**dict(vocab_size=2000, hidden=H, layers=layers, heads=heads, ffn=F, max_pos=512, type_vocab=2,
                                num_labels=labels), **kw})


LENS = [0, 1, 2, 147, 0, 255, 256, 257, 512, 0]     # empty sequences first, in the middle and last
# case: (config, weight scale, sequence lengths, c).  c bounds both the max and the RMS ratio to fp32's error: twice the
# worst ratio over the six outputs measured on an H100 (DESIGN.md section 2), rounded up.
CASES = {
    "MiniLM-L6": (_preset("all-MiniLM-L6-v2"), 1.0, LENS, 28),
    "MiniLM-L6 x4": (_preset("ms-marco-MiniLM-L-6-v2"), 4.0, LENS, 22),
    "bge-base": (_preset("bge-base-en-v1.5"), 1.0, LENS, 34),
    # bge-large / mxbai-embed-large: E1 at K = 4096, N = 3072 / 4096; 24 layers of accumulated error
    "H1024 dh64 L24": (_cfg(1024, 16, 4096, 24, 1), 1.0, LENS, 60),
    "H1024 dh32": (_cfg(1024, 32, 4096, 2, 3), 1.0, LENS, 52),
    # QKV 21 tiles, LayerNorm at 7 values per lane, F != 4H
    "H896 dh64 F2688": (_cfg(896, 14, 2688, 2, 1), 1.0, LENS, 46),
    # d_h 64 at the smallest H, F = 5 tiles
    "H128 dh64 F640": (_cfg(128, 2, 640, 2, 2), 4.0, LENS, 20),
    # the layers == 0 branch; one layer, where the CLS path's last layer is also its first
    "L0": (_cfg(384, 12, 1536, 0, 2), 1.0, LENS, 8),
    "L1": (_cfg(384, 12, 1536, 1, 1), 4.0, LENS, 20),
    # positions up to max_pos - 1 (a sequence of exactly max_pos); pair type ids 1 clamped to the only row, 0
    "max_pos 128, type_vocab 1": (_cfg(384, 6, 1536, 2, 1, max_pos=128, type_vocab=1), 4.0, [0, 1, 2, 127, 0, 128, 100, 0],
                                  16),
}


def _batch(lens, vocab, seed):
    rng = np.random.default_rng(seed)
    ids = np.concatenate([np.r_[101, rng.integers(104, vocab, max(n - 2, 0)), 102][:n] for n in lens] +
                         [np.zeros(0, np.int64)]).astype(np.int32)
    typ = np.concatenate([np.r_[np.zeros(n // 3, np.int32), np.ones(n - n // 3, np.int32)] for n in lens])
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    return ids, typ, cu, max(lens)


def _gpu_outputs(enc, ids, typ, cu, mx):
    out = {"hidden": enc.hidden_tokens(ids, typ, cu, mx)}
    for mode in ("mean", "cls"):
        out[mode] = enc.embed_tokens(ids, typ, cu, mx, mode, False)
        out[mode + "_norm"] = enc.embed_tokens(ids, typ, cu, mx, mode, True)
    out["logits"] = enc.classify_tokens(ids, typ, cu, mx)
    torch.cuda.synchronize()
    return out


def _fp32_outputs(w32, cfg, ids, typ, cu):
    """bert_ref's padded fp32 forward on the device (type ids clamped, as the kernels clamp them; bert_ref indexes the
    table directly).  Rows of empty sequences are left out of err_32 (their padded CLS row is not defined there)."""
    lens = np.diff(cu)
    S = int(lens.max())
    I = np.zeros((len(lens), S), np.int64); M = np.zeros_like(I); Ty = np.zeros_like(I)
    for b, n in enumerate(lens):
        I[b, :n] = ids[cu[b]:cu[b + 1]]
        Ty[b, :n] = np.clip(typ[cu[b]:cu[b + 1]], 0, cfg.type_vocab - 1)
        M[b, :n] = 1
    ocfg = bert_ref.BertCfg(**asdict(cfg))
    with torch.no_grad():
        h = bert_ref.bert_encoder_forward(w32, ocfg, *(torch.from_numpy(a) for a in (I, M, Ty)), device="cuda")
        mask = torch.from_numpy(M).cuda()
        out = {"hidden": torch.cat([h[b, :n] for b, n in enumerate(lens)])}
        for mode in ("mean", "cls"):
            out[mode] = bert_ref.pool(h, mask, mode)
            out[mode + "_norm"] = bert_ref.l2_normalize(out[mode])
        out["logits"] = bert_ref.classifier_head(w32, h)
    return {k: v.double() for k, v in out.items()}


def _err(d):
    d = d.abs()
    return float(d.max()), float(d.pow(2).mean().sqrt())


_STACK = {}


def _stack(case):
    """(encoder, weights on the device, batch, GPU outputs, float64 outputs on the split weights, fp32 outputs)"""
    if case not in _STACK:
        from ragmeup_b200.encoder import BertEncoder
        _STACK.clear()                                   # one set of weights at a time (24 x 1024 x 4096 is 1.2 GB)
        cfg, scale, lens, _ = CASES[case]
        w = synthetic_bert_weights(cfg, seed=31 + cfg.layers + cfg.hidden, with_head=True, scale=scale)
        enc = BertEncoder(cfg, w, with_head=True)
        wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
        del w
        w32 = {k: ref.split_weight(v).float() if k.endswith(ref.GEMM_WEIGHTS) else v for k, v in wd.items()}
        batch = _batch(lens, cfg.vocab_size, seed=len(case))
        ids, typ, cu, mx = batch
        got = _gpu_outputs(enc, *batch)
        want = ref.encoder_stack_ref(wd, cfg, ids, typ, cu, "split", device="cuda")
        f32 = _fp32_outputs(w32, cfg, ids, typ, cu)
        _STACK[case] = (enc, wd, batch, got, want, f32)
    return _STACK[case]


@pytest.mark.parametrize("case", list(CASES))
def test_encoder_matches_float64_forward_on_split_weights(cuda, case):
    enc, wd, (ids, typ, cu, mx), got, want, f32 = _stack(case)
    c = CASES[case][3]
    nonempty = torch.from_numpy(np.diff(cu) > 0).cuda()
    report, fails = [], []
    for name in OUTPUTS:
        g, w_, f = got[name].double(), want[name], f32[name]
        assert torch.isfinite(g).all(), f"{name}: not finite"
        rows = slice(None) if name == "hidden" else nonempty
        gmax, grms = _err(g - w_)
        fmax, frms = _err(f[rows] - w_[rows])
        mag_max, mag_rms = float(w_.abs().max()), float(w_.pow(2).mean().sqrt())
        rmax, rrms = gmax / max(fmax, 1e-300), grms / max(frms, 1e-300)
        report.append(f"{name} max {gmax:.3g} / fp32 {fmax:.3g} = {rmax:.3g}, rms {grms:.3g} / {frms:.3g} = {rrms:.3g}")
        if gmax > c * fmax + FLOOR * U * mag_max or grms > c * frms + FLOOR * U * mag_rms:
            fails.append(f"{name}: max {gmax:.3g} (ratio {rmax:.3g}), rms {grms:.3g} (ratio {rrms:.3g})")
    print(f"\nstack {case}:\n  " + "\n  ".join(report))
    # an empty sequence: zero embeddings, logits W_c tanh(b_p) + b_c (the same wherever it sits)
    empty = ~nonempty
    for name in ("mean", "mean_norm", "cls", "cls_norm"):
        assert (got[name][empty] == 0).all(), name
    e = got["logits"][empty]
    assert (e == e[0]).all()
    _check_bit_identities(enc, ids, typ, cu, got)
    assert not fails, f"{case}: beyond {c} x fp32's error: " + "; ".join(fails)


def _bits(t):
    t = torch.as_tensor(t).contiguous()
    return t.view(torch.int32).cpu().numpy()


def _assert_same(a, b, what):
    ga, gb = _bits(a), _bits(b)
    if not np.array_equal(ga, gb):
        rows = sorted(set(np.nonzero(ga != gb)[0].tolist()))
        pytest.fail(f"{what}: not bit-identical in rows {rows[:16]} ({len(rows)} rows)")


def _check_bit_identities(enc, ids, typ, cu, got):
    """embed_host / classify_host equal the device entry points bit for bit; each sequence alone equals its rows in the
    batch (hidden, embeddings, logits)"""
    for mode in ("mean", "cls"):
        for norm in (False, True):
            key = mode + ("_norm" if norm else "")
            _assert_same(torch.from_numpy(enc.embed_host(ids, typ, cu, mode, norm)), got[key], f"embed_host {key}")
    _assert_same(torch.from_numpy(enc.classify_host(ids, typ, cu)), got["logits"], "classify_host")
    lens = np.diff(cu)
    for b in sorted({int(np.argmax(lens)), 1, 3, len(lens) - 2}):
        t0, t1 = int(cu[b]), int(cu[b + 1])
        if t1 == t0:
            continue
        one = _gpu_outputs(enc, ids[t0:t1], typ[t0:t1], np.array([0, t1 - t0], np.int32), t1 - t0)
        _assert_same(one["hidden"], got["hidden"][t0:t1], f"sequence {b} alone: hidden")
        for name in OUTPUTS[1:]:
            _assert_same(one[name][0], got[name][b], f"sequence {b} alone: {name}")


def test_sequence_longer_than_max_pos_is_refused(cuda):
    from ragmeup_b200._lib import RmuError
    enc = _stack("max_pos 128, type_vocab 1")[0]
    ids, typ, cu, _ = _batch([129], enc.cfg.vocab_size, 0)
    with pytest.raises(RmuError, match="max_position_embeddings"):
        enc.embed_tokens(ids, typ, cu, 129)


# ---------------------------------------------------------------------------------------------- batch limits
SMALL = _cfg(128, 4, 256, 2, 2, vocab_size=1000, max_pos=128)
_SMALL = {}


def _small_encoder():
    """(encoder, its weights on the device)"""
    if not _SMALL:
        from ragmeup_b200.encoder import BertEncoder
        w = synthetic_bert_weights(SMALL, seed=41, with_head=True, scale=4.0)
        _SMALL["enc"] = BertEncoder(SMALL, w, with_head=True)
        _SMALL["w"] = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    return _SMALL["enc"], _SMALL["w"]


@pytest.mark.parametrize("B", [65535, 65536, 70000])
def test_batches_past_the_65535_sequence_grid_limit(cuda, B):
    """attention puts the sequence in gridDim.y (at most 65 535) and runs larger batches in slices: every sequence, on
    either side of a slice edge, equals itself alone bit for bit and the float64 forward on a sample"""
    enc, wd = _small_encoder()
    rng = np.random.default_rng(B)
    lens = rng.integers(0, 4, B)
    lens[65532] = 0
    sample = sorted({0, 1, 65533, 65534, min(65535, B - 1), min(65536, B - 1), B - 2, B - 1,
                     *rng.integers(0, B, 6).tolist()})
    for s in sample:
        lens[s] = 1 + s % 3                               # sampled sequences are not empty
    ids, typ, cu, mx = _batch(lens.tolist(), SMALL.vocab_size, B)
    got = _gpu_outputs(enc, ids, typ, cu, mx)
    for s in sample:
        t0, t1 = int(cu[s]), int(cu[s + 1])
        sub = (ids[t0:t1], typ[t0:t1], np.array([0, t1 - t0], np.int32))
        one = _gpu_outputs(enc, *sub, t1 - t0)
        _assert_same(one["hidden"], got["hidden"][t0:t1], f"sequence {s} alone: hidden")
        for name in OUTPUTS[1:]:
            _assert_same(one[name][0], got[name][s], f"sequence {s} alone: {name}")
        want = ref.encoder_stack_ref(wd, SMALL, *sub, "split", device="cuda")
        for name in OUTPUTS:
            g = got["hidden"][t0:t1] if name == "hidden" else got[name][s:s + 1]
            assert float((g.double() - want[name]).abs().max()) < 1e-5 * (1 + float(want[name].abs().max())), \
                f"sequence {s}: {name} differs from the float64 forward"
    empty = torch.from_numpy(np.diff(cu) == 0).cuda()
    assert (got["mean"][empty] == 0).all() and (got["cls"][empty] == 0).all()


def test_encode_tensor_of_65536_empty_texts(cuda):
    """65 536 empty texts are 65 536 two-token sequences, exactly MAX_TOKENS_PER_CALL, so one call: every row equals the
    embedding of one empty text"""
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.encoder import MAX_TOKENS_PER_CALL
    emb = HuggingFaceEmbeddings(model_name="synthetic:tiny")
    assert 2 * 65536 == MAX_TOKENS_PER_CALL
    out = emb.encode_tensor([""] * 65536)
    one = emb.encode_tensor([""])
    assert out.shape == (65536, emb.config.hidden)
    _assert_same(out, one.expand(65536, -1), "encode_tensor([''] * 65536)")


def _one_token_words(tok, vocab_size):
    from ragmeup_b200.tokenizer import synthetic_vocab
    words = [w for w in synthetic_vocab(vocab_size) if w.isalpha() and len(w) > 1][:400]
    return [w for w, e in zip(words, tok.encode_batch(words, add_special_tokens=False)) if len(e.ids) == 1]


def _texts(words, counts, rng):
    return [" ".join(rng.choice(words, n)) for n in counts]


@pytest.mark.parametrize("extra", [0, 1])
def test_python_chunking_at_max_tokens_per_call(cuda, extra):
    """T = MAX_TOKENS_PER_CALL and one token past it through encode_tensor, embed_host and score_tensor: every row is
    bit-identical to the same text (pair) encoded alone, in input order across the chunk edge"""
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.encoder import MAX_TOKENS_PER_CALL, BertEncoder
    emb = HuggingFaceEmbeddings(model_name="synthetic:tiny")
    assert emb.max_seq_length == 64
    rng = np.random.default_rng(extra)
    words = _one_token_words(emb.tokenizer, emb.config.vocab_size)
    assert len(words) > 50
    n = MAX_TOKENS_PER_CALL // 64
    # 64-token texts (62 words); with extra, the last full text is one token short and an empty text (2 tokens) follows
    counts = [62] * n if not extra else [62] * (n - 1) + [61, 0]
    texts = _texts(words, counts, rng)
    ids, typ, cu = emb._ragged(texts)
    assert int(cu[-1]) == MAX_TOKENS_PER_CALL + extra
    chunks = list(BertEncoder._chunks(cu, MAX_TOKENS_PER_CALL))
    assert len(chunks) == 1 + extra
    check = sorted({0, 1, n // 2, n - 2, n - 1, len(texts) - 1})
    out = emb.encode_tensor(texts)
    host = emb.client.embed_host(ids, typ, cu, emb.pooling, emb.normalize)
    for i in check:
        alone = emb.encode_tensor([texts[i]])[0]
        _assert_same(out[i], alone, f"encode_tensor row {i}")
        _assert_same(torch.from_numpy(host[i]), alone, f"embed_host row {i}")
    ce = HuggingFaceCrossEncoder(model_name="synthetic:tiny")
    assert ce.max_length == 64
    # pairs [CLS] a [SEP] b [SEP]: 30 + 31 words = 64 tokens; with extra, one pair of 63 and an empty pair of 3
    pc = [(30, 31)] * n if not extra else [(30, 31)] * (n - 1) + [(30, 29), (0, 0)]
    pairs = list(zip(_texts(words, [a for a, _ in pc], rng), _texts(words, [b for _, b in pc], rng)))
    pids, _, pcu = ce._pairs([p[0] for p in pairs], [p[1] for p in pairs])
    assert int(pcu[-1]) == MAX_TOKENS_PER_CALL + extra
    scores = ce.score_tensor(pairs)
    for i in check:
        _assert_same(scores[i:i + 1], ce.score_tensor([pairs[i]]), f"score_tensor row {i}")


def _all_outputs(enc, batch):
    o = _gpu_outputs(enc, *batch)
    return [o[k].clone() for k in OUTPUTS]


def test_workspace_growth_keeps_results(cuda):
    """one handle through small, large and small T, and through B past seq_cap (1024) with T small: every result is
    bit-identical to a fresh handle's"""
    from ragmeup_b200.encoder import BertEncoder
    w = synthetic_bert_weights(SMALL, seed=41, with_head=True, scale=4.0)
    rng = np.random.default_rng(3)
    small = _batch(rng.integers(1, 60, 12).tolist(), SMALL.vocab_size, 1)
    large = _batch(rng.integers(1, 129, 400).tolist(), SMALL.vocab_size, 2)            # ~26 000 tokens
    lens = np.zeros(3000, np.int64)
    lens[rng.choice(3000, 300, replace=False)] = rng.integers(1, 4, 300)              # B = 3000, T < 1024
    many = _batch(lens.tolist(), SMALL.vocab_size, 3)
    assert int(many[2][-1]) < 1024 < len(lens)
    fresh = {}
    for name, batch in (("small", small), ("large", large), ("many", many)):
        fresh[name] = _all_outputs(BertEncoder(SMALL, w, with_head=True), batch)
    for seq in (("small", "large", "small"), ("small", "many", "small")):
        h = BertEncoder(SMALL, w, with_head=True)
        for name in seq:
            batch = {"small": small, "large": large, "many": many}[name]
            for k, a, b in zip(OUTPUTS, _all_outputs(h, batch), fresh[name]):
                _assert_same(a, b, f"{' -> '.join(seq)}: {name} {k}")


def test_max_seqlen_at_max_pos_is_bit_identical(cuda):
    """max_seqlen may be anything from the longest sequence to max_pos: more row blocks exit at once, and the key
    blocks (multiples of 32) keep their order"""
    enc, _ = _small_encoder()
    rng = np.random.default_rng(4)
    ids, typ, cu, mx = _batch(rng.integers(0, 41, 200).tolist(), SMALL.vocab_size, 4)
    a = _gpu_outputs(enc, ids, typ, cu, mx)
    b = _gpu_outputs(enc, ids, typ, cu, SMALL.max_pos)
    for k in OUTPUTS:
        _assert_same(a[k], b[k], f"max_seqlen {mx} vs {SMALL.max_pos}: {k}")
