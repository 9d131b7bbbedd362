"""Attention provenance on the GPU: the span kernels against float64 on given planes (rmu_debug_attention_spans), the
Llama stack against the float64 forward, compute_attention end to end against the oracle for Llama and Qwen3, and the
refusals that name the model."""
from __future__ import annotations

import gc
import math
from dataclasses import asdict, replace

import numpy as np
import pytest
import torch

from oracle import encoder_kernels_ref as ref
from oracle import decoder_attention_ref as da
from oracle import qwen3_ref
from ragmeup_b200.weights import DECODER_PRESETS, LlamaConfig, Qwen3Config, resolve_decoder, synthetic_llama_weights

pytestmark = pytest.mark.gpu
STACK_RATIO = 32.0          # as the Qwen3 stack: the GPU's error may be at most this multiple of the fp32 forward's


@pytest.fixture(autouse=True)
def _release_torch_cache():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _lib():
    from ragmeup_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------------- the span kernels
def _spans_cases(T, rng):
    """overlapping, nested, repeated, empty (start == end and end < start), one-token, touching T - 1, whole-sequence
    spans, and enough of them to need two chunks of column spans"""
    s = [(0, T), (0, 0), (T // 2, T // 2), (min(3, T), max(0, T - 7)), (T - 1, T), (max(0, T - 5), T), (0, 1)]
    a, b = T // 5, (3 * T) // 4
    s += [(a, b), (a, b), (a + T // 10, b - T // 10), (T // 3, T), (b, min(T, b + 1))]
    while len(s) < 41:
        x = int(rng.integers(0, T))
        s.append((x, int(rng.integers(x, min(T, x + 300) + 1))))
    return s


def _ref_span_mass(planes, T, heads, kv, spans):
    """float64: the causal base-2 softmax of the joined planes, summed over each (row span, column span) pair"""
    x = planes[0].double() + planes[1].double()
    G, n = heads // kv, len(spans)
    out = torch.zeros(n, n, dtype=torch.float64, device="cuda")
    lo = torch.tensor([min(max(s, 0), T) for s, _ in spans])
    hi = torch.maximum(torch.tensor([min(max(e, 0), T) for _, e in spans]), lo)
    cols = torch.zeros(n, T, dtype=torch.float64, device="cuda")
    for b in range(n):
        cols[b, lo[b]:hi[b]] = 1.0
    for r0 in range(0, T, 2048):
        r1 = min(T, r0 + 2048)
        live = [a for a in range(n) if lo[a] < r1 and hi[a] > r0 and lo[a] < hi[a]]
        if not live:
            continue
        mask = torch.arange(T, device="cuda")[None, :] > torch.arange(r0, r1, device="cuda")[:, None]
        for h in range(heads):
            q = x[r0:r1, h * 128:(h + 1) * 128]
            k = x[:, (heads + h // G) * 128:(heads + h // G + 1) * 128]
            s = (q @ k.T).masked_fill(mask, float("-inf")) * math.log(2.0)
            p = s.softmax(-1) @ cols.T                       # [rows, n]: each row's mass per column span
            for a in live:
                i0, i1 = max(lo[a], r0) - r0, min(hi[a], r1) - r0
                out[a] += p[i0:i1].sum(0)
    return out


def _sparse_spans(T):
    """spans in the middle and at the end only, none over the whole sequence: most row blocks meet no span, so the
    span kernels skip them (as they skip a thread's system prompt)"""
    return [(T // 3, T // 3 + 100), (T // 3 + 40, T // 3 + 50), (T // 2, T // 2), (T // 2 + 7, T // 2 + 8),
            ((2 * T) // 3, (2 * T) // 3 + 130), (T - 97, T), (T - 20, T - 5)]


@pytest.mark.parametrize("T,heads,kv,sparse", [(1, 4, 4, False), (17, 8, 2, False), (300, 32, 8, False),
                                               (300, 4, 4, False), (4097, 32, 8, False), (4097, 8, 2, False),
                                               (20000, 4, 4, False), (4097, 32, 8, True), (4097, 4, 4, True),
                                               (20000, 8, 2, True)])
def test_span_kernel_matches_float64(T, heads, kv, sparse):
    rng = np.random.default_rng(T + heads)
    NH = heads + 2 * kv
    x = (0.42 * rng.standard_normal((T, NH * 128))).astype(np.float32)     # base-2 scores of spread ~2
    planes = [torch.from_numpy(p).cuda() for p in ref.split_f16(x)]
    spans = _sparse_spans(T) if sparse else _spans_cases(T, rng)
    d_spans = torch.tensor(spans, dtype=torch.int32, device="cuda")
    out = torch.full((len(spans), len(spans)), float("nan"), dtype=torch.float64, device="cuda")
    _lib().check(_lib().lib().rmu_debug_attention_spans(planes[0].data_ptr(), planes[1].data_ptr(), T, heads, kv,
                                                         d_spans.data_ptr(), len(spans), out.data_ptr(), None),
                 "rmu_debug_attention_spans")
    torch.cuda.synchronize()
    want = _ref_span_mass(planes, T, heads, kv, spans)
    size = torch.tensor([max(0, min(e, T) - min(max(s, 0), T)) for s, e in spans], dtype=torch.float64, device="cuda")
    tol = 1e-5 * heads * size[:, None]
    err = (out - want).abs()
    assert bool((err <= tol).all()), float((err - tol).max())
    if not sparse:   # a column span of the whole sequence takes every row's full mass
        assert bool(((out[:, 0] - heads * size).abs() <= 1e-5 * heads * size).all())
    # the same inputs give the same bits
    again = torch.empty_like(out)
    _lib().check(_lib().lib().rmu_debug_attention_spans(planes[0].data_ptr(), planes[1].data_ptr(), T, heads, kv,
                                                         d_spans.data_ptr(), len(spans), again.data_ptr(), None),
                 "rmu_debug_attention_spans")
    assert torch.equal(out, again)


# ------------------------------------------------------------------------------------------------- the Llama stack
def _llama_errors(cfg, w, lens, seed):
    from ragmeup_b200.encoder import BertEncoder
    enc = BertEncoder(cfg, w, with_head=False)
    rng = np.random.default_rng(seed)
    seqs = [rng.integers(0, cfg.vocab_size, n).tolist() for n in lens]
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    ids = np.concatenate([np.asarray(s, np.int32) for s in seqs])
    got = enc.hidden_tokens(ids, None, cu, max(lens)).double()
    W64, W32 = qwen3_ref.weights(w, torch.float64, "cuda"), qwen3_ref.weights(w, torch.float32, "cuda")
    want = torch.cat([da.hidden(W64, cfg, s, torch.float64, qk_norm=False) for s in seqs])
    f32 = torch.cat([da.hidden(W32, cfg, s, torch.float32, qk_norm=False) for s in seqs]).double()
    e_gpu, e_32 = (got - want).abs(), (f32 - want).abs()
    return (float(e_gpu.max()), float(e_gpu.pow(2).mean().sqrt())), (float(e_32.max()), float(e_32.pow(2).mean().sqrt()))


@pytest.mark.parametrize("shape", ["tiny-llama", "llama-3.1-8b-2-layers"])
def test_llama_stack_matches_float64_forward(shape):
    if shape == "tiny-llama":
        cfg, lens = LlamaConfig(**asdict(DECODER_PRESETS["tiny-llama"])), [1, 17, 129, 600]
    else:   # two layers of the 8B shape (a small vocabulary: the table is not what is tested)
        cfg, lens = replace(LlamaConfig(**asdict(DECODER_PRESETS["llama-3.1-8b"])), layers=2, vocab_size=1000), [2048]
    w = synthetic_llama_weights(cfg, seed=11, scale=2.0)
    (gm, gr), (fm, fr) = _llama_errors(cfg, w, lens, 12)
    print(f"\n{shape}: gpu max {gm:.3g} rms {gr:.3g}; fp32 max {fm:.3g} rms {fr:.3g}; ratios {gm / fm:.3g} {gr / fr:.3g}")
    assert gm <= STACK_RATIO * fm and gr <= STACK_RATIO * fr


# ------------------------------------------------------------------------------------------------- end to end
WORDS = ["system", "user", "assistant", "question", "answer", "document", "the", "capital", "of", "France", "is",
         "Paris", "river", "Seine", "flows", "through", "Berlin", "Germany", "context"]


def _chat(n_docs, filler):
    docs = [f"document {i}: the river Seine flows through Paris " + "the " * (i * filler) + f"{i}" for i in range(n_docs)]
    query = "question: what is the capital of France"
    answer = "answer: the capital of France is Paris"
    thread = ("<|im_start|>system\nanswer the question from the context\n" + "\n".join(docs) + "<|im_end|>\n"
              f"<|im_start|>user\n{query}<|im_end|>\n<|im_start|>assistant\n{answer}<|im_end|>\n")
    return thread, query, docs, answer


@pytest.mark.parametrize("model", ["synthetic:tiny-llama", "synthetic:tiny-qwen3"])
@pytest.mark.parametrize("include", ["True", "False"])
def test_compute_attention_matches_oracle(monkeypatch, model, include):
    from transformers import PreTrainedTokenizerFast
    from ragmeup_b200 import provenance
    from ragmeup_b200.tokenizer import build_byte_bpe
    monkeypatch.setenv("attribute_include_query", include)
    tok = PreTrainedTokenizerFast(tokenizer_object=build_byte_bpe(WORDS))
    thread, query, docs, answer = _chat(5, 7)
    got = provenance.compute_attention(model, tok, thread, query, docs, answer)
    dec = provenance._decoder(model)
    assert provenance._decoder(model) is dec                      # uploaded once per process
    ids = tok.encode(thread, add_special_tokens=False)
    W = qwen3_ref.weights(resolve_decoder(model)[1], torch.float64, "cuda")
    A = da.last_attention(W, dec.cfg, ids, qk_norm=isinstance(dec.cfg, Qwen3Config)).cpu().numpy()
    enc = lambda t: tok.encode(t, add_special_tokens=False)       # noqa: E731
    want = da.attention_scores(A, ids, enc(query), enc(answer), [enc(d) for d in docs], include_query=include == "True")
    assert len(got) == len(docs) and all(isinstance(g, np.float64) for g in got)
    np.testing.assert_allclose(got, want, rtol=1e-3)


def test_refusals_name_the_model():
    from ragmeup_b200 import _lib, provenance
    dec = provenance.DecoderAttention("synthetic:tiny-llama")
    with pytest.raises(ValueError, match="synthetic:tiny-llama.*max_position_embeddings"):
        dec.span_mass(list(range(dec.cfg.max_pos + 1)), [(0, 1)])
    big = provenance.DecoderAttention("synthetic:tiny-llama:0:30000")   # projections ~600: activations leave fp16
    with pytest.raises(_lib.RmuError, match="synthetic:tiny-llama:0:30000.*65504"):
        big.span_mass(list(range(64)), [(0, 8), (8, 64)])


def _oracle_mass(dec, ids, spans):
    W = qwen3_ref.weights(resolve_decoder(dec.name)[1], torch.float64, "cuda")
    A = da.last_attention(W, dec.cfg, ids, qk_norm=isinstance(dec.cfg, Qwen3Config))
    return torch.stack([torch.stack([A[:, a0:a1, b0:b1].sum() for b0, b1 in spans]) for a0, a1 in spans]).cpu().numpy()


def test_span_mass_skips_rows_after_a_dense_call():
    """one handle, its span workspace reused: a call whose spans cover the whole thread, then one whose spans leave most
    row blocks out, against the float64 forward's attention"""
    from ragmeup_b200 import provenance
    dec = provenance.DecoderAttention("synthetic:tiny-llama:5")
    ids = np.random.default_rng(21).integers(0, dec.cfg.vocab_size, 700).tolist()
    heads = dec.cfg.heads
    for spans in ([(0, 700), (0, 350), (350, 700), (100, 600)], _sparse_spans(700)):
        got, want = dec.span_mass(ids, spans), _oracle_mass(dec, ids, spans)
        size = np.array([max(0, e - s) for s, e in spans], dtype=np.float64)
        assert (np.abs(got - want) <= 1e-4 * heads * size[:, None]).all(), np.abs(got - want).max()


def test_llama_golden(golden_dir, monkeypatch):
    """tests/golden/llama.npz (the float64 oracle): the hidden state, the span masses and both score settings"""
    import importlib.util
    import os
    from ragmeup_b200 import provenance
    path = os.path.join(golden_dir, "make_golden_llama.py")
    spec = importlib.util.spec_from_file_location("make_golden_llama", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g = np.load(os.path.join(golden_dir, "llama.npz"))
    dec = provenance.DecoderAttention(mod.MODEL)
    ids = g["ids"]
    T, heads = len(ids), dec.cfg.heads
    h = dec.encoder.hidden_tokens(ids, None, np.array([0, T], np.int32), T).cpu().numpy()
    err = np.abs(h - g["hidden"]).max()
    print(f"\nllama golden: hidden max |delta| {err:.3g}")
    assert err <= 5e-4
    spans = [tuple(s) for s in g["spans"].tolist()]
    size = np.array([e - s for s, e in spans], dtype=np.float64)
    assert (np.abs(dec.span_mass(ids.tolist(), spans) - g["mass"]) <= 1e-4 * heads * size[:, None]).all()
    text, query, docs, answer = mod.thread()
    tok = mod.tokenizer()
    assert tok.encode(text, add_special_tokens=False) == ids.tolist()
    for setting, key in (("True", "scores_q"), ("False", "scores_noq")):
        monkeypatch.setenv("attribute_include_query", setting)
        got = provenance.compute_attention(dec, tok, text, query, docs, answer)
        np.testing.assert_allclose(got, g[key], rtol=1e-3, equal_nan=True)
