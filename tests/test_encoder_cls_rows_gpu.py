"""GPU: the classifier head and CLS pooling run the encoder's last layer on the CLS rows only (K and V for every token,
the rest of the layer for row cu[b] of each sequence).  Every kernel computes a row from that row alone, so the outputs
must be bit-identical to the full stack's.

Reference, through public entry points: rmu_encoder_hidden (every layer on every row) -> rmu_debug_split_planes ->
rmu_debug_cls_head / rmu_debug_pool (CLS) with the original cu.  The heads read hi + lo in fp32, so as long as
join(split(h)) == h bit for bit (checked first, up to the sign of a zero, see _assert_identical) this is exactly what
the full stack's heads computed.  A zero's sign cannot reach a logit (the head's first fmaf from +0 returns +0 for
either sign), so the logits are compared strictly.
"""
from dataclasses import asdict

import numpy as np
import pytest
import torch

from ragmeup_b200.weights import PRESETS, BertConfig, synthetic_bert_weights

pytestmark = pytest.mark.gpu
POOL_CLS = 1

_ENCODERS = {}


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _encoder(shape, layers, num_labels):
    """(encoder, device weights of the head); shape "minilm" is the full ms-marco-MiniLM-L-6 preset, "dh32" / "dh64"
    are H 384 / 768 with 12 heads and a small vocabulary"""
    from ragmeup_b200.encoder import BertEncoder
    key = (shape, layers, num_labels)
    if key not in _ENCODERS:
        if shape == "minilm":
            cfg = BertConfig(**asdict(PRESETS["ms-marco-MiniLM-L-6-v2"][0]))
        else:
            H = 384 if shape == "dh32" else 768
            cfg = BertConfig(vocab_size=2000, hidden=H, layers=layers, heads=12, ffn=4 * H, max_pos=512)
        cfg.num_labels = num_labels
        w = synthetic_bert_weights(cfg, seed=7 + layers + num_labels, with_head=True, scale=4.0)
        head = {k: torch.from_numpy(w[k]).cuda() for k in ("pooler.dense.weight", "pooler.dense.bias", "classifier.weight",
                                                            "classifier.bias")}
        _ENCODERS[key] = (BertEncoder(cfg, w, with_head=True), head)
    return _ENCODERS[key]


def _bits(t):
    return t.contiguous().view(torch.int32).cpu().numpy()


def _assert_identical(got, want, what, zero_sign=True):
    """bit-identical; with zero_sign=False -0 and +0 count as the same: a hidden value in (-2^-25, 0) is stored as the
    planes (-0, -0), joins to -0, and re-splits into (-0, +0), which joins to +0.  Every other value survives the
    re-split bit for bit."""
    if not zero_sign:
        got, want = got + 0.0, want + 0.0
    g, w = _bits(got), _bits(want)
    if not np.array_equal(g, w):
        rows = sorted(set(np.nonzero(g != w)[0].tolist()))
        pytest.fail(f"{what}: not bit-identical to the full stack in rows {rows[:16]} ({len(rows)} rows)")


def _batch(lens, typed, vocab, seed):
    rng = np.random.default_rng(seed)
    lens = [int(n) for n in lens]
    ids = np.concatenate([rng.integers(104, vocab, n) for n in lens] + [np.zeros(0, np.int64)]).astype(np.int32)
    typ = rng.integers(0, 2, ids.size).astype(np.int32) if typed else None
    cu = np.r_[0, np.cumsum(lens)].astype(np.int32)
    return ids, typ, cu, max(lens)


def _reference(enc, head, ids, typ, cu, mx):
    """full stack: last hidden state [T, H], its split planes, the head's logits and the CLS embeddings"""
    L = _lib()
    lib = L.lib()
    H, nl = enc.cfg.hidden, enc.cfg.num_labels
    B = len(cu) - 1
    h = enc.hidden_tokens(ids, typ, cu, mx)
    hi = torch.empty(h.shape, dtype=torch.float16, device="cuda")
    lo = torch.empty_like(hi)
    L.check(lib.rmu_debug_split_planes(h.data_ptr(), h.numel(), hi.data_ptr(), lo.data_ptr(), L.stream_ptr()), "split")
    back = torch.empty_like(h)
    L.check(lib.rmu_debug_join_planes(hi.data_ptr(), lo.data_ptr(), h.numel(), back.data_ptr(), L.stream_ptr()), "join")
    _assert_identical(back, h, "join(split(hidden))", zero_sign=False)
    cu_d = torch.from_numpy(cu).cuda()
    logits = torch.empty((B, nl), dtype=torch.float32, device="cuda")
    L.check(lib.rmu_debug_cls_head(hi.data_ptr(), lo.data_ptr(), cu_d.data_ptr(), B, H, nl,
                                   head["pooler.dense.weight"].data_ptr(), head["pooler.dense.bias"].data_ptr(),
                                   head["classifier.weight"].data_ptr(), head["classifier.bias"].data_ptr(),
                                   logits.data_ptr(), L.stream_ptr()), "cls_head")
    emb = {}
    for norm in (0, 1):
        e = torch.empty((B, H), dtype=torch.float32, device="cuda")
        L.check(lib.rmu_debug_pool(hi.data_ptr(), lo.data_ptr(), cu_d.data_ptr(), B, H, POOL_CLS, norm, e.data_ptr(),
                                   L.stream_ptr()), "pool")
        emb[norm] = e
    torch.cuda.synchronize()
    return h, logits, emb


# (encoder shape, layers, num_labels, sequence lengths, type ids present)
CASES = {
    # the headline's rerank call: 800 pairs x 147 tokens through the full MiniLM-L6 cross-encoder
    "minilm_bench_800x147": ("minilm", 6, 1, [147] * 800, True),
    # one key block, block edges, the 256-key super-block and past it, up to max_position_embeddings
    "dh32_lengths": ("dh32", 2, 3, [1, 2, 16, 17, 147, 255, 256, 257, 512], True),
    "dh64_lengths": ("dh64", 2, 1, [1, 2, 16, 17, 147, 255, 256, 257, 512], True),
    # empty sequences first, in the middle and last; no type ids
    "dh32_empty_seqs": ("dh32", 2, 1, [0, 0, 5, 0, 147, 1, 0, 0], False),
    "dh64_empty_seqs": ("dh64", 2, 3, [0, 33, 0, 2, 0], False),
    # more sequences than tokens
    "dh32_b_gt_t": ("dh32", 2, 3, [0, 0, 1, 0, 0, 2, 0, 0, 0, 1, 0], True),
    "dh64_b_gt_t": ("dh64", 1, 1, [0, 1, 0, 0, 0], False),
    # B at the edges of E1's 128-row tiles (the compact rows)
    "dh32_b1": ("dh32", 2, 1, [40], True),
    "dh32_b127": ("dh32", 2, 1, np.random.default_rng(1).integers(1, 40, 127), True),
    "dh32_b128": ("dh32", 2, 3, np.random.default_rng(2).integers(1, 40, 128), False),
    "dh32_b129": ("dh32", 2, 1, np.random.default_rng(3).integers(0, 40, 129), True),
    "dh64_b129": ("dh64", 2, 3, np.random.default_rng(4).integers(1, 40, 129), True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_cls_rows_last_layer_is_bit_identical(cuda, case):
    shape, layers, nl, lens, typed = CASES[case]
    enc, head = _encoder(shape, layers, nl)
    ids, typ, cu, mx = _batch(lens, typed, enc.cfg.vocab_size, seed=len(lens) + 17 * layers)
    B = len(cu) - 1
    h, want_logits, want_emb = _reference(enc, head, ids, typ, cu, mx)

    _assert_identical(enc.classify_tokens(ids, typ, cu, mx), want_logits, "rmu_encoder_classify")
    _assert_identical(torch.from_numpy(enc.classify_host(ids, typ, cu)), want_logits, "rmu_encoder_classify_host")
    for norm in (0, 1):
        got = enc.embed_tokens(ids, typ, cu, mx, "cls", bool(norm))
        _assert_identical(got, want_emb[norm], f"rmu_encoder_embed (CLS, normalize={norm})", zero_sign=False)
    # unnormalised CLS embeddings are the hidden state's CLS rows (zero for an empty sequence)
    raw = enc.embed_tokens(ids, typ, cu, mx, "cls", False)
    nonempty = torch.from_numpy(np.nonzero(np.diff(cu) > 0)[0]).cuda()
    rows = h[torch.from_numpy(cu[:-1]).cuda()[nonempty].long()]
    _assert_identical(raw[nonempty], rows, "CLS embedding vs hidden[cu[b]]")
    empty = torch.from_numpy(np.nonzero(np.diff(cu) == 0)[0]).cuda()
    assert (raw[empty] == 0).all()
    assert B == len(lens)
