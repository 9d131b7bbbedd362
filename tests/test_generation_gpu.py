"""Generation on the GPU decoder: decode attention and the sampler against float64 (rmu_debug_attention_decode,
rmu_debug_sample), rmu_decoder_generate against the float64 oracle's greedy tokens and sampled distribution, its stop
rules and refusals, and the handle compute_attention and generation share."""
from __future__ import annotations

import ctypes as C
import gc
import math
from dataclasses import replace

import numpy as np
import pytest
import torch

import make_golden_generate as mg
from oracle import decoder_attention_ref as da
from oracle import generation_ref as gref
from ragmeup_b200.weights import (DECODER_PRESETS, PRESETS, LlamaConfig, Qwen3Config, synthetic_llama_weights,
                                  synthetic_qwen3_weights)

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release_torch_cache():
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    yield


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _split(x):
    hi = x.to(torch.float16)
    lo = (x - hi.float()).to(torch.float16)
    return hi, lo


def _sampling(do_sample=False, temperature=1.0, top_k=50, top_p=1.0, penalty=1.0, eos=()):
    L = _lib()
    return L.SamplingC(int(do_sample), temperature, top_p, penalty, top_k, len(eos), (C.c_int32 * L.MAX_EOS)(*eos))


# ------------------------------------------------------------------------------------------------- decode attention
@pytest.mark.parametrize("G", [1, 2, 4, 8])
@pytest.mark.parametrize("n", [1, 7, 255, 256, 257, 1000, 4097, 32768])
def test_attention_decode_matches_float64(G, n):
    L = _lib()
    kv_heads = 2 if G < 8 else 1
    heads, cap = G * kv_heads, n + 5
    g = torch.Generator(device="cuda").manual_seed(n * 31 + G)
    q = torch.randn(heads, 128, device="cuda", generator=g) * (1.4426950408889634 / math.sqrt(128))
    k = torch.randn(kv_heads, cap, 128, device="cuda", generator=g) * 2.0
    v = torch.randn(kv_heads, cap, 128, device="cuda", generator=g)
    qh, ql = _split(q)
    kh, kl = _split(k)
    vh, vl = _split(v)
    kv = torch.stack([kh, kl, vh, vl]).contiguous()
    ws = torch.empty(heads * ((n + 63) // 64) * 130, device="cuda")
    outs = []
    for _ in range(2):
        ch = torch.empty(heads * 128, dtype=torch.float16, device="cuda")
        cl = torch.empty_like(ch)
        L.check(L.lib().rmu_debug_attention_decode(qh.data_ptr(), ql.data_ptr(), kv.data_ptr(), heads, kv_heads, cap, n,
                                                   ws.data_ptr(), ws.numel(), ch.data_ptr(), cl.data_ptr(),
                                                   L.stream_ptr()), "rmu_debug_attention_decode")
        torch.cuda.synchronize()
        outs.append((ch.clone(), cl.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    got = (outs[0][0].double() + outs[0][1].double()).view(heads, 128)
    qd = qh.double() + ql.double()
    kd = (kh.double() + kl.double())[:, :n]
    vd = (vh.double() + vl.double())[:, :n]
    kr, vr = kd.repeat_interleave(G, 0), vd.repeat_interleave(G, 0)
    s = torch.einsum("hd,hjd->hj", qd, kr) * math.log(2.0)
    ref = torch.einsum("hj,hjd->hd", s.softmax(-1), vr)
    err = (got - ref).abs().max().item()
    assert err < 2e-5, err


def test_attention_decode_refusals():
    L = _lib()
    ws = torch.empty(16, device="cuda")
    x = torch.empty(4096, dtype=torch.float16, device="cuda")
    p = x.data_ptr()
    f = L.lib().rmu_debug_attention_decode
    assert f(p, p, p, 3, 2, 8, 4, ws.data_ptr(), 4096, p, p, None) == -3
    assert f(p, p, p, 2, 2, 8, 9, ws.data_ptr(), 4096, p, p, None) == -1
    assert f(p, p, p, 2, 2, 8, 4, ws.data_ptr(), 10, p, p, None) == -1


# ------------------------------------------------------------------------------------------------- the sampler
def _run_sample(x, seen, s, u):
    L = _lib()
    V = x.size
    d = torch.as_tensor(x, dtype=torch.float32, device="cuda").contiguous()
    bits = np.zeros((V + 31) // 32, dtype=np.uint32)
    for i in set(seen):
        bits[i >> 5] |= np.uint32(1 << (i & 31))
    pres = torch.as_tensor(bits.view(np.int32), device="cuda")
    tok = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(L.lib().rmu_debug_sample(d.data_ptr(), V, pres.data_ptr(), C.byref(s), u, tok.data_ptr(), L.stream_ptr()),
            "rmu_debug_sample")
    torch.cuda.synchronize()
    t = int(tok.item())
    assert (pres.cpu().numpy().view(np.uint32)[t >> 5] >> (t & 31)) & 1
    return t, d.cpu().numpy()


@pytest.mark.parametrize("V", [1000, 128256, 151936])
def test_sampler_greedy_ties_and_penalty(V):
    rng = np.random.default_rng(V)
    x = rng.standard_normal(V).astype(np.float32)
    x[[17, 400, V - 3]] = 9.0                                  # a three-way tie: the lowest id wins
    t, _ = _run_sample(x, [], _sampling(), 0.0)
    assert t == 17
    seen = [17, 400, 5, 6]
    x[5], x[6] = 8.5, -9.5                                     # penalised positive and negative logits
    for pen in (1.3, 0.7):
        want = gref.repetition_penalty(x.astype(np.float64), seen, pen)
        t, got = _run_sample(x, seen, _sampling(penalty=pen), 0.0)
        assert np.allclose(got, want, rtol=1e-6, atol=0)
        assert t == gref.greedy(want.astype(np.float32))


@pytest.mark.parametrize("V", [1000, 128256, 151936])
def test_sampler_draws_match_oracle(V):
    rng = np.random.default_rng(V + 1)
    x = (3.0 * rng.standard_normal(V)).astype(np.float32)
    x[rng.choice(V, 40, replace=False)] = np.float32(np.sort(x)[-30])    # ties at and around the k-th value
    for k, p, temp in ((1, 1.0, 1.0), (50, 0.9, 0.7), (256, 0.95, 1.3), (20, 1.0, 1.0), (256, 0.3, 1.0)):
        xt = (x.astype(np.float32) / np.float32(temp)).astype(np.float64)
        c = gref.kept(xt, gref.candidates(xt, k), p)
        w = np.exp(xt[c] - xt[c[0]])
        edges = np.cumsum(w) / w.sum()
        for u in np.linspace(0.0, 0.999, 23):
            if np.min(np.abs(edges - u)) < 1e-5:
                continue                                         # a CDF edge: float32 and float64 may disagree
            t, _ = _run_sample(x, [], _sampling(True, temp, k, p), float(u))
            assert t == gref.draw(xt, k, p, float(u)), (k, p, temp, u)


def test_sampler_top_k_tie_cap():
    V = 1000
    x = np.zeros(V, dtype=np.float32)
    x[900] = 1.0
    # 999 logits tie at the k-th value: the candidates are id 900 and the 255 lowest tied ids
    c = gref.candidates(x.astype(np.float64), 5)
    assert len(c) == 256 and c[0] == 900 and list(c[1:4]) == [0, 1, 2]
    for u in (0.1, 0.5, 0.99):
        t, _ = _run_sample(x, [], _sampling(True, 1.0, 5, 1.0), u)
        assert t == gref.draw(x.astype(np.float64), 5, 1.0, u)


def test_sampler_top_p_boundary():
    # probabilities 0.5, 0.3, 0.2: top_p 0.5 keeps one, 0.75 two, 0.85 three
    x = np.log(np.array([0.2, 0.5, 0.3] + [1e-30] * 125)).astype(np.float32)
    for p, n in ((0.45, 1), (0.75, 2), (0.85, 3)):
        assert len(gref.kept(x.astype(np.float64), gref.candidates(x.astype(np.float64), 3), p)) == n
        seen = {_run_sample(x, [], _sampling(True, 1.0, 3, p), u)[0] for u in np.linspace(0, 0.999, 40)}
        assert len(seen) == n


# ------------------------------------------------------------------------------------------------- generate
def _decoder(kind, vocab=1024, scale=6.0, seed=3, max_pos=8192):
    """a tiny decoder (make_golden_generate.model) on the GPU with its LM head attached"""
    from ragmeup_b200.encoder import BertEncoder
    cfg, w, lm = mg.model(kind, vocab=vocab, scale=scale, seed=seed, max_pos=max_pos)
    enc = BertEncoder(cfg, w, with_head=False)
    L = _lib()
    enc._check(L.lib().rmu_decoder_set_lm_head(enc._h, lm.ctypes.data), "rmu_decoder_set_lm_head")
    return cfg, w, lm, enc


def _generate(enc, ids, s, seed, max_new, logits=None):
    L = _lib()
    prompt = np.ascontiguousarray(ids, dtype=np.int32)
    out = np.zeros(max_new, dtype=np.int32)
    n = C.c_int32(0)
    rc = L.lib().rmu_decoder_generate(enc._h, prompt.ctypes.data, len(prompt), C.byref(s), seed, max_new,
                                      out.ctypes.data, C.byref(n), None if logits is None else logits.ctypes.data,
                                      L.stream_ptr())
    return rc, out[:n.value].tolist()


@pytest.mark.parametrize("kind", mg.KINDS)
def test_generate_matches_fixture(kind, golden_dir):
    import os
    z = np.load(os.path.join(golden_dir, "generate.npz"))
    cfg, w, lm, enc = _decoder(kind)
    for i in range(len(mg.PROMPT_LENS)):
        ids = z[f"{kind}_{i}_prompt"].tolist()
        logits = np.zeros((mg.STEPS, cfg.vocab_size), np.float32)
        rc, got = _generate(enc, ids, _sampling(penalty=mg.PENALTY), 0, mg.STEPS, logits)
        assert rc == 0 and got == z[f"{kind}_{i}_tokens"].tolist()
        ref = z[f"{kind}_{i}_logits"]
        err = np.abs(logits[:mg.LOGIT_STEPS] - ref).max() / np.abs(ref).max()
        assert err < 2e-5, err


@pytest.mark.parametrize("kind", mg.KINDS)
def test_decode_step_logits_match_prefill(kind):
    """step t's logits (decode attention over the cache) against a prefill of the T + t tokens plus the LM head"""
    cfg, w, lm, enc = _decoder(kind)
    ids = np.random.default_rng(9).integers(0, cfg.vocab_size, 300).tolist()
    N = 20
    steps = np.zeros((N, cfg.vocab_size), np.float32)
    rc, toks = _generate(enc, ids, _sampling(penalty=1.2), 0, N, steps)
    assert rc == 0 and len(toks) == N
    for t in (1, 2, 7, 19):
        one = np.zeros((1, cfg.vocab_size), np.float32)
        rc, _ = _generate(enc, ids + toks[:t], _sampling(), 0, 1, one)
        assert rc == 0
        # two fp32 paths with different summation orders (SIMT decode attention, mma.sync prefill): the bound is the
        # fixture's against float64; a wrong cache row or position moves the logits by O(1)
        err = np.abs(steps[t] - one[0]).max() / np.abs(one[0]).max()
        assert err < 2e-5, (t, err)


def test_llama_8b_shape_two_layers_against_float64():
    """two layers of the Llama-3.1-8B shape (hidden 4096, 32 / 8 heads, F 14336, vocabulary 128 256): a 2 048-token
    prefill and 16 steps; every step's logits against the float64 forward of the same tokens"""
    from ragmeup_b200.encoder import BertEncoder
    cfg = replace(DECODER_PRESETS["llama-3.1-8b"], layers=2)
    w = synthetic_llama_weights(cfg, seed=4)
    lm = (0.02 * np.random.default_rng(5).standard_normal((cfg.vocab_size, cfg.hidden))).astype(np.float32)
    enc = BertEncoder(cfg, w, with_head=False)
    L = _lib()
    enc._check(L.lib().rmu_decoder_set_lm_head(enc._h, lm.ctypes.data), "rmu_decoder_set_lm_head")
    T, N = 2048, 16
    ids = np.random.default_rng(6).integers(0, cfg.vocab_size, T).tolist()
    got = np.zeros((N + 1, cfg.vocab_size), np.float32)
    rc, toks = _generate(enc, ids, _sampling(), 0, N + 1, got)
    assert rc == 0 and len(toks) == N + 1
    del enc
    gc.collect()
    torch.cuda.empty_cache()
    wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    h = da.hidden(wd, cfg, ids + toks[:N], torch.float64, qk_norm=False)[T - 1:]
    ref = (h @ torch.from_numpy(lm).cuda().double().T).cpu().numpy()
    del wd, h
    err = np.abs(got - ref).max() / np.abs(ref).max()
    assert err < 1e-4, err
    for t in range(N + 1):
        top2 = np.sort(ref[t])[-2:]
        if top2[1] - top2[0] > 1e-3 * np.abs(ref).max():
            assert toks[t] == int(np.argmax(ref[t])), t


@pytest.mark.parametrize("kind", mg.KINDS)
def test_generate_greedy_matches_oracle(kind):
    cfg, w, lm, enc = _decoder(kind)
    rng = np.random.default_rng(5)
    for T in (1, 9, 300):
        ids = rng.integers(0, cfg.vocab_size, T).tolist()
        rc, got = _generate(enc, ids, _sampling(penalty=1.2), 0, 12)
        assert rc == 0
        want = gref.generate(w, lm, cfg, ids, 12, qk_norm=kind == "qwen3", penalty=1.2)
        assert got == want, (T, got, want)
    # the cache allocation is reused, and a shorter call after a longer one gives the same tokens
    rc, again = _generate(enc, ids[:9], _sampling(penalty=1.2), 0, 12)
    rc2, first = _generate(enc, ids[:9], _sampling(penalty=1.2), 0, 12)
    assert rc == rc2 == 0 and again == first


@pytest.mark.parametrize("kind", mg.KINDS)
def test_generate_sampled_matches_oracle_and_repeats(kind):
    cfg, w, lm, enc = _decoder(kind, scale=1.0)
    ids = list(range(3, 40))
    s = _sampling(True, 0.8, 50, 0.9, 1.1)
    rc, a = _generate(enc, ids, s, 1234, 6)
    rc2, b = _generate(enc, ids, s, 1234, 6)
    assert rc == rc2 == 0 and a == b
    want = gref.generate(w, lm, cfg, ids, 6, qk_norm=kind == "qwen3", do_sample=True, temp=0.8, k=50, p=0.9,
                         penalty=1.1, seed=1234)
    assert a == want


def test_generate_first_token_frequencies():
    from scipy.stats import chisquare
    cfg, w, lm, enc = _decoder("llama", scale=1.0)
    lm = lm * 0.05                                             # a flat distribution: many tokens in play
    L = _lib()
    from ragmeup_b200.encoder import BertEncoder
    enc = BertEncoder(cfg, w, with_head=False)
    enc._check(L.lib().rmu_decoder_set_lm_head(enc._h, np.ascontiguousarray(lm).ctypes.data), "set_lm_head")
    ids = [5, 6, 7, 8]
    x = gref.temperature(gref.logits(w, lm, cfg, ids, False), 1.0)
    prob = gref.probabilities(x, 8, 1.0)
    counts = np.zeros(cfg.vocab_size)
    N = 2000
    for seed in range(N):
        rc, t = _generate(enc, ids, _sampling(True, 1.0, 8, 1.0), seed, 1)
        assert rc == 0
        counts[t[0]] += 1
    sup = prob > 0
    assert counts[~sup].sum() == 0
    assert chisquare(counts[sup], prob[sup] * N).pvalue > 1e-3


def test_generate_stops_and_refusals():
    cfg, w, lm, enc = _decoder("llama", max_pos=20)
    ids = list(range(1, 11))
    rc, full = _generate(enc, ids, _sampling(), 0, 5)
    assert rc == 0 and len(full) == 5                           # max_new_tokens
    rc, cut = _generate(enc, ids, _sampling(eos=(full[2],)), 0, 5)
    assert rc == 0 and cut == full[:full.index(full[2]) + 1]     # the eos token is returned
    rc, longest = _generate(enc, ids, _sampling(), 0, 50)
    assert rc == 0 and len(longest) == 10                      # prompt and output fill max_pos = 20
    assert _generate(enc, list(range(20)), _sampling(), 0, 5)[0] == -1
    assert _generate(enc, ids, _sampling(True, 1.0, 0), 0, 5)[0] == -3
    assert _generate(enc, ids, _sampling(True, 1.0, 257), 0, 5)[0] == -3
    assert _generate(enc, ids, _sampling(True, 0.0, 5), 0, 5)[0] == -1
    assert _generate(enc, [cfg.vocab_size], _sampling(), 0, 5)[0] == -1
    L = _lib()
    assert L.lib().rmu_decoder_set_lm_head(enc._h, lm.ctypes.data) == -1       # a second head


def test_generate_range_error():
    cfg, w, lm, enc = _decoder("llama", scale=3000.0)
    rc, _ = _generate(enc, list(range(1, 30)), _sampling(), 0, 3)
    assert rc == -4


def test_pipeline_end_to_end_and_shared_handle(tmp_path):
    """HuggingFacePipeline around a transformers pipeline on a tiny saved snapshot returns the text that pipeline
    returns on the CPU, greedy; the reply is found as _extract_reply finds it; compute_attention on the same model
    then runs on the same decoder handle"""
    from transformers import AutoModelForCausalLM, AutoTokenizer, pipeline
    from ragmeup_b200 import provenance
    from ragmeup_b200.llms import HuggingFacePipeline
    mg.save_chat_snapshot(str(tmp_path))
    model = AutoModelForCausalLM.from_pretrained(str(tmp_path)).eval()
    tok = AutoTokenizer.from_pretrained(str(tmp_path))
    pipe = pipeline(model=model, tokenizer=tok, task="text-generation", temperature=0.6, repetition_penalty=1.1,
                    return_full_text=True, max_new_tokens=16, do_sample=False)
    llm = HuggingFacePipeline(pipeline=pipe)
    for prompt in ("w5 w6 w7 w8 w9 w10 w11 " + mg.ASSISTANT, " ".join(f"w{4 + (i * 37) % 250}" for i in range(120)) +
                   " " + mg.ASSISTANT):
        with torch.no_grad():
            want = pipe(prompt)[0]["generated_text"]
        got = llm.invoke(prompt)
        assert got == want
        assert got[got.rindex(mg.ASSISTANT) + len(mg.ASSISTANT):] == want[len(prompt):]
    n = len(provenance._DECODERS)
    dec = provenance._decoder(model)
    assert dec._lm_head                                          # attached by the generation above
    scores = provenance.compute_attention(model, tok, "w5 w6 w7 w8 w9 w10 w11", "w5 w6", ["w7 w8 w9"], "w10 w11")
    assert len(scores) == 1 and np.isfinite(scores[0])
    assert provenance._decoder(model) is dec and len(provenance._DECODERS) == n
