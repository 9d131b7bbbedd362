"""Prompt-lookup decoding on the GPU decoder (rmu_decoder_generate_lookup, rmu_debug_generate_drafts): every call
returns rmu_decoder_generate's tokens and logits bit for bit, on split and NF4 handles, greedy and sampled, whatever the
drafts; the drafts are really used (the pass counts the accept rule implies); the verify pass's sampler rows one at a
time against rmu_debug_sample; a verify pass that leaves the fp16 range falls back to the single-row step; and the
Python entry points."""
from __future__ import annotations

import ctypes as C
import gc
import math

import numpy as np
import pytest
import torch

import make_golden_generate as mg
from oracle import generation_ref as gref

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


def _handle(kind, weights="split", max_pos=8192, cfg_w_lm=None):
    from ragmeup_b200.encoder import BertEncoder
    cfg, w, lm = cfg_w_lm or mg.model(kind, max_pos=max_pos)
    enc = BertEncoder(cfg, w, with_head=False)
    L = _lib()
    if weights == "nf4":
        enc._check(L.lib().rmu_decoder_quantize_nf4(enc._h, L.stream_ptr()), "rmu_decoder_quantize_nf4")
    enc._check(L.lib().rmu_decoder_set_lm_head(enc._h, np.ascontiguousarray(lm).ctypes.data), "set_lm_head")
    return cfg, w, lm, enc


def _sampling(do_sample=False, temp=1.0, k=50, p=1.0, penalty=1.0, eos=()):
    L = _lib()
    return L.SamplingC(int(do_sample), temp, p, penalty, k, len(eos), (C.c_int32 * L.MAX_EOS)(*eos))


def _plain(enc, V, ids, s, seed, max_new):
    L = _lib()
    prompt = np.ascontiguousarray(ids, dtype=np.int32)
    out = np.zeros(max_new, dtype=np.int32)
    logits = np.full((max_new, V), np.nan, dtype=np.float32)
    n = C.c_int32(0)
    rc = L.lib().rmu_decoder_generate(enc._h, prompt.ctypes.data, len(prompt), C.byref(s), seed, max_new,
                                      out.ctypes.data, C.byref(n), logits.ctypes.data, L.stream_ptr())
    assert rc == 0, L.lib().rmu_last_error()
    return out[:n.value].tolist(), logits


def _drafted(enc, V, ids, s, seed, max_new, drafts, k):
    """rmu_debug_generate_drafts -> (rc, tokens, logits [max_new, V], passes)"""
    L = _lib()
    prompt = np.ascontiguousarray(ids, dtype=np.int32)
    d = np.ascontiguousarray(drafts, dtype=np.int32)
    assert len(d) == max_new
    out = np.zeros(max_new, dtype=np.int32)
    logits = np.full((max_new, V), np.nan, dtype=np.float32)
    n, passes = C.c_int32(0), C.c_int32(-1)
    rc = L.lib().rmu_debug_generate_drafts(enc._h, prompt.ctypes.data, len(prompt), C.byref(s), seed, max_new,
                                           d.ctypes.data, k, out.ctypes.data, C.byref(n), logits.ctypes.data,
                                           C.byref(passes), L.stream_ptr())
    return rc, out[:n.value].tolist(), logits, passes.value


def _lookup(enc, V, ids, s, seed, max_new, k, ngram=2):
    L = _lib()
    prompt = np.ascontiguousarray(ids, dtype=np.int32)
    out = np.zeros(max_new, dtype=np.int32)
    logits = np.full((max_new, V), np.nan, dtype=np.float32)
    n, passes = C.c_int32(0), C.c_int32(-1)
    rc = L.lib().rmu_decoder_generate_lookup(enc._h, prompt.ctypes.data, len(prompt), C.byref(s), seed, max_new, k,
                                             ngram, out.ctypes.data, C.byref(n), logits.ctypes.data, C.byref(passes),
                                             L.stream_ptr())
    assert rc == 0, L.lib().rmu_last_error()
    return out[:n.value].tolist(), logits, passes.value


def _same(a, b):
    """tokens and logits bit for bit; the rows after the last token untouched (NaN) in both"""
    assert a[0] == b[0]
    assert np.array_equal(a[1].view(np.int32), b[1].view(np.int32))


def _check(enc, V, ids, s, seed, max_new, drafts, k, passes=None):
    want = _plain(enc, V, ids, s, seed, max_new)
    rc, toks, logits, n_pass = _drafted(enc, V, ids, s, seed, max_new, drafts, k)
    assert rc == 0, _lib().lib().rmu_last_error()
    _same((toks, logits), want)
    if passes is not None:
        assert n_pass == passes, (k, n_pass, passes)
    return want[0], n_pass


def _wrong_every(toks, j, V, max_new):
    d = list(toks) + [0] * (max_new - len(toks))
    return [(t + 1) % V if m % j == 0 else t for m, t in enumerate(d)]


SETTINGS = [
    _sampling(penalty=1.3),
    _sampling(True, 0.8, 40, 0.9, 1.3),
]


@pytest.mark.parametrize("weights", ["split", "nf4"])
@pytest.mark.parametrize("kind", mg.KINDS)
def test_injected_drafts_equal_plain(kind, weights):
    cfg, w, lm, enc = _handle(kind, weights)
    V, max_new = cfg.vocab_size, 40
    rng = np.random.default_rng(1)
    prompt = rng.integers(0, V, 37).tolist()
    for i, s in enumerate(SETTINGS):
        seed = 100 + i
        toks, _ = _plain(enc, V, prompt, s, seed, max_new)
        assert len(toks) == max_new
        for k in (1, 2, 7, 15):
            # every draft right: ceil((n - 1) / (k + 1)) passes after the prefill; every draft wrong: n - 1
            _check(enc, V, prompt, s, seed, max_new, toks, k, passes=math.ceil((max_new - 1) / (k + 1)))
            _check(enc, V, prompt, s, seed, max_new, _wrong_every(toks, 1, V, max_new), k, passes=max_new - 1)
            for j in (2, 5):
                _check(enc, V, prompt, s, seed, max_new, _wrong_every(toks, j, V, max_new), k)
            _check(enc, V, prompt, s, seed, max_new, rng.integers(0, V, max_new).tolist(), k)
        # an EOS inside an accepted run ends the call there
        eos = toks[11]
        s_eos = _sampling(bool(s.do_sample), s.temperature, s.top_k, s.top_p, s.repetition_penalty, eos=(eos,))
        got, _ = _check(enc, V, prompt, s_eos, seed, max_new, toks, 7)
        assert got == toks[:toks.index(eos) + 1]
        # max_new_tokens reached inside what a pass of 15 drafts would cover
        for m in (2, 3, 10, 17):
            _check(enc, V, prompt, s, seed, m, toks[:m], 15, passes=math.ceil((m - 1) / 16))


@pytest.mark.parametrize("weights", ["split", "nf4"])
def test_injected_drafts_near_max_pos(weights):
    """a prompt ending a few positions before max_pos = 64: passes are capped so that no row reaches past it"""
    cfg, w, lm, enc = _handle("llama", weights, max_pos=64)
    V = cfg.vocab_size
    rng = np.random.default_rng(2)
    for T in (55, 60, 62, 63):
        prompt = rng.integers(0, V, T).tolist()
        for s in SETTINGS:
            toks, _ = _plain(enc, V, prompt, s, 3, 20)
            assert len(toks) == 64 - T
            d = toks + [0] * (20 - len(toks))
            _check(enc, V, prompt, s, 3, 20, d, 15, passes=math.ceil((len(toks) - 1) / 16))
            _check(enc, V, prompt, s, 3, 20, _wrong_every(toks, 2, V, 20), 7)


def _copy_model(kind):
    """a decoder whose greedy next token is perm(last token): projections near zero (the residual is the token's
    embedding), LM head row perm(t) along embedding t, so a reply continues any run t, perm(t), perm(perm(t)), ... of
    the prompt"""
    cfg, w, _ = mg.model(kind, scale=0.05)
    emb = w["embed_tokens.weight"]
    perm = np.random.default_rng(7).permutation(cfg.vocab_size)
    lm = np.zeros_like(emb)
    lm[perm] = emb * (8.0 / np.linalg.norm(emb, axis=1, keepdims=True))
    return (cfg, w, lm), perm


@pytest.mark.parametrize("weights", ["split", "nf4"])
@pytest.mark.parametrize("kind", mg.KINDS)
def test_ngram_lookup_end_to_end(kind, weights):
    """rmu_decoder_generate_lookup equals rmu_decoder_generate on prompts with repeated spans; on the copying decoder,
    whose greedy reply repeats a run of the prompt, it takes fewer passes than tokens"""
    cfg, w, lm, enc = _handle(kind, weights)
    V = cfg.vocab_size
    rng = np.random.default_rng(3)
    span = rng.integers(0, V, 12).tolist()
    prompts = [span + rng.integers(0, V, 5).tolist() + span + span[:4],
               (span[:3] * 6) + rng.integers(0, V, 9).tolist() + span[:3],
               rng.integers(0, V, 30).tolist()]
    for prompt in prompts:
        for s in SETTINGS:
            want = _plain(enc, V, prompt, s, 9, 24)
            for k, ngram in ((1, 1), (4, 2), (10, 3), (20, 2)):
                toks, logits, _ = _lookup(enc, V, prompt, s, 9, 24, k, ngram)
                _same((toks, logits), want)
    del enc
    cfg_w_lm, perm = _copy_model(kind)
    cfg, w, lm, enc = _handle(kind, weights, cfg_w_lm=cfg_w_lm)
    run = [5]
    for _ in range(40):
        run.append(int(perm[run[-1]]))
    prompt = run[:40] + rng.integers(0, V, 6).tolist() + run[:10]
    s = _sampling()
    want = _plain(enc, V, prompt, s, 0, 24)
    assert want[0][:20] == run[10:30]                         # the reply repeats the prompt's run
    toks, logits, passes = _lookup(enc, V, prompt, s, 0, 24, 7)
    _same((toks, logits), want)
    assert passes < len(toks) - 1
    assert passes <= math.ceil(23 / 8) + 1


@pytest.mark.parametrize("sampled", [False, True])
def test_sampler_verify_rows_equal_one_row_launches(sampled):
    """rmu_debug_sample_verify_rows: row j (presence = base | drafts 1 .. j, u = philox(seed, step0 + j)) equals
    rmu_debug_sample on that row with those bits set by hand: token, processed logits and bits; the base is not
    written.  Draft id 4 000 is absent from the base and tops every row: greedy, a row that ignored the draft bits
    would choose it, with the penalty it loses to id 10."""
    L = _lib()
    V, M, seed, step0 = 5000, 6, 2 ** 63 + 11, 9
    words = (V + 31) // 32
    g = torch.Generator(device="cuda").manual_seed(int(sampled))
    logits = torch.randn(M, V, device="cuda", generator=g)
    base = torch.randint(0, 2 ** 31 - 1, (words,), dtype=torch.int32, device="cuda", generator=g)
    ids_h = [17, 33, 4000, 33, 2500, 4999]                     # the pending token, then the drafts
    for b in (4000, 10):
        base[b // 32] &= ~(1 << (b % 32))
    logits[:, 4000] = 9.0
    logits[:, 10] = 8.0
    ids = torch.tensor(ids_h, dtype=torch.int32, device="cuda")
    s = _sampling(True, 0.7, 40, 0.9, 1.3) if sampled else _sampling(penalty=1.3)
    lg, pr = logits.clone(), base.clone()
    rows = torch.full((M, words), -1, dtype=torch.int32, device="cuda")
    tok = torch.full((M,), -1, dtype=torch.int32, device="cuda")
    L.check(L.lib().rmu_debug_sample_verify_rows(lg.data_ptr(), V, M, pr.data_ptr(), ids.data_ptr(), seed, step0,
                                                 C.byref(s), rows.data_ptr(), tok.data_ptr(), L.stream_ptr()),
            "sample_verify_rows")
    torch.cuda.synchronize()
    assert torch.equal(pr, base)
    for j in range(M):
        l1, p1 = logits[j].clone(), base.clone()
        for d in ids_h[1:j + 1]:
            p1[d // 32] |= 1 << (d % 32)
        t1 = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        u = gref.philox_uniform(seed, step0 + j)
        L.check(L.lib().rmu_debug_sample(l1.data_ptr(), V, p1.data_ptr(), C.byref(s), float(u), t1.data_ptr(),
                                         L.stream_ptr()), "sample")
        torch.cuda.synchronize()
        assert int(tok[j]) == int(t1[0]), j
        assert torch.equal(lg[j].view(torch.int32), l1.view(torch.int32)) and torch.equal(rows[j], p1), j
    if not sampled:
        assert [int(t) for t in tok[:4]] == [4000, 4000, 10, 10]


def test_range_fallback_returns_the_plain_tokens():
    """a token z whose embedding row is past fp32's range (its activations are NaN, outside fp16) never enters the
    plain greedy run; fed as a rejected draft it raises the range flag, and the pass is redone as a single-row step:
    RMU_OK and the plain tokens and logits.  A prompt holding z still fails with RMU_ERR_RANGE."""
    cfg, w, lm = mg.model("llama")
    V = cfg.vocab_size
    prompt = np.random.default_rng(4).integers(0, V, 20).tolist()
    _, _, _, enc = _handle("llama", cfg_w_lm=(cfg, w, lm))
    clean, _ = _plain(enc, V, prompt, _sampling(), 0, 16)
    del enc
    z = next(t for t in range(V) if t not in prompt and t not in clean)
    w = dict(w)
    w["embed_tokens.weight"] = w["embed_tokens.weight"].copy()
    w["embed_tokens.weight"][z] = np.inf
    _, _, _, enc = _handle("llama", cfg_w_lm=(cfg, w, lm))
    want = _plain(enc, V, prompt, _sampling(), 0, 16)
    assert want[0] == clean and z not in want[0]
    for drafts in ([z] * 16, [clean[m] if m % 3 else z for m in range(16)]):
        for k in (1, 4, 15):
            rc, toks, logits, _ = _drafted(enc, V, prompt, _sampling(), 0, 16, drafts, k)
            assert rc == 0, _lib().lib().rmu_last_error()
            _same((toks, logits), want)
    rc, _, _, _ = _drafted(enc, V, prompt + [z], _sampling(), 0, 4, clean[:4], 3)
    assert rc == -4


def test_refusals_on_a_handle():
    cfg, w, lm, enc = _handle("llama", max_pos=64)
    L = _lib()
    V = cfg.vocab_size
    ids = np.arange(1, 6, dtype=np.int32)
    out = np.zeros(4, np.int32)
    n, passes = C.c_int32(), C.c_int32()
    s = _sampling()
    lookup = L.lib().rmu_decoder_generate_lookup
    args = (out.ctypes.data, C.byref(n), None, C.byref(passes), None)
    assert lookup(enc._h, ids.ctypes.data, 5, C.byref(s), 0, 4, 3, 2, *args) == 0
    assert lookup(enc._h, ids.ctypes.data, 5, C.byref(s), 0, 4, -1, 2, *args) == -1
    assert lookup(enc._h, ids.ctypes.data, 5, C.byref(s), 0, 4, 3, 0, *args) == -1
    big = np.arange(64, dtype=np.int32)
    assert lookup(enc._h, big.ctypes.data, 64, C.byref(s), 0, 4, 3, 2, *args) == -1      # T >= max_pos
    d = np.full(4, V, np.int32)
    assert L.lib().rmu_debug_generate_drafts(enc._h, ids.ctypes.data, 5, C.byref(s), 0, 4, d.ctypes.data, 3,
                                             *args) == -1                                  # a draft id out of range
    d[:] = 0
    assert L.lib().rmu_debug_generate_drafts(enc._h, ids.ctypes.data, 5, C.byref(s), 0, 4, d.ctypes.data, -1,
                                             *args) == -1


def test_decoder_attention_and_pipeline(tmp_path, monkeypatch):
    """DecoderAttention.generate with prompt_lookup_num_tokens equals plain generate; HuggingFacePipeline with
    RMU_PROMPT_LOOKUP_TOKENS set returns the text it returns without it"""
    from transformers import AutoModelForCausalLM, AutoTokenizer, pipeline
    from ragmeup_b200 import llms, provenance
    mg.save_chat_snapshot(str(tmp_path))
    dec = provenance.DecoderAttention(str(tmp_path))
    rng = np.random.default_rng(8)
    span = rng.integers(0, dec.cfg.vocab_size, 10).tolist()
    ids = span + rng.integers(0, dec.cfg.vocab_size, 4).tolist() + span[:5]
    for kw in (dict(), dict(do_sample=True, temperature=0.7, top_k=30, top_p=0.9, repetition_penalty=1.1, seed=4)):
        want = dec.generate(ids, 20, **kw)
        for k, g in ((3, 2), (10, 1), (40, 3)):
            assert dec.generate(ids, 20, prompt_lookup_num_tokens=k, max_matching_ngram_size=g, **kw) == want
    del dec
    model = AutoModelForCausalLM.from_pretrained(str(tmp_path)).eval()
    tok = AutoTokenizer.from_pretrained(str(tmp_path))
    pipe = pipeline(model=model, tokenizer=tok, task="text-generation", temperature=0.6, repetition_penalty=1.1,
                    return_full_text=True, max_new_tokens=16, do_sample=False)
    llm = llms.HuggingFacePipeline(pipeline=pipe)
    prompt = "w5 w6 w7 w8 w9 w5 w6 w7 w8 w9 w5 w6 " + mg.ASSISTANT
    monkeypatch.delenv(llms.PROMPT_LOOKUP_ENV, raising=False)
    want = llm.invoke(prompt)
    monkeypatch.setenv(llms.PROMPT_LOOKUP_ENV, "10")
    assert llm.invoke(prompt) == want
