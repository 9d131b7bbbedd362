"""Speculative decoding with a draft model on the GPU decoder (rmu_decoder_generate_assisted): every call returns
rmu_decoder_generate's tokens and logits bit for bit, whatever the draft computes; a draft with the target's own
weights has every draft kept in the pass count the loop's caps give; any mix of split and NF4 handles runs; the edges
(one or two new tokens, a prompt near max_pos, a draft with a shorter max_pos, a draft whose activations leave the fp16
range); the refusals on live handles; concurrent calls; and the Python entry points."""
from __future__ import annotations

import ctypes as C
import gc
import threading
from dataclasses import replace

import numpy as np
import pytest
import torch

import make_golden_generate as mg

pytestmark = pytest.mark.gpu

CONSTANT, HEURISTIC = 0, 1
TARGET = "synthetic:tiny-llama:0"


@pytest.fixture(autouse=True)
def _release_torch_cache():
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    yield


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _handle(name, weights="split", max_pos=None, layers=None, lm_head=True):
    """a decoder handle of the synthetic model ``name``, split or NF4, with its LM head.  The tiny presets' vocabulary
    of 1000 becomes 1024, which the LM head GEMM's 128-row tile takes; ``max_pos`` replaces the preset's; ``layers``
    builds the first layers of a large preset one layer at a time (SyntheticDecoderLayers)."""
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import (LlamaConfig, SyntheticDecoderLayers, decoder_config, synthetic_llama_weights,
                                      synthetic_qwen3_weights)
    L = _lib()
    parts = name.split(":")
    seed = int(parts[2]) if len(parts) > 2 else 0
    scale = float(parts[3]) if len(parts) > 3 else 1.0
    cfg = decoder_config(name)
    if cfg.vocab_size % 128:
        cfg = replace(cfg, vocab_size=1024)
    if max_pos:
        cfg = replace(cfg, max_pos=max_pos)
    if layers is not None:
        cfg = replace(cfg, layers=layers)
        src = SyntheticDecoderLayers(cfg, seed=seed, scale=scale)
        if weights == "nf4":
            enc = BertEncoder.nf4_decoder(src)
        else:
            w = dict(src.globals())
            for l in range(layers):
                w.update(src.layer(l))
            enc = BertEncoder(cfg, w, with_head=False)
    else:
        w = (synthetic_llama_weights(cfg, seed=seed, scale=scale) if isinstance(cfg, LlamaConfig)
             else synthetic_qwen3_weights(cfg, seed=seed, scale=scale))
        enc = BertEncoder(cfg, w, with_head=False)
        if weights == "nf4":
            enc._check(L.lib().rmu_decoder_quantize_nf4(enc._h, L.stream_ptr()), "rmu_decoder_quantize_nf4")
    if lm_head:
        lm = np.ascontiguousarray(0.02 * scale * np.random.default_rng([seed, 1]).standard_normal(
            (cfg.vocab_size, cfg.hidden)), dtype=np.float32)
        enc._check(L.lib().rmu_decoder_set_lm_head(enc._h, lm.ctypes.data), "rmu_decoder_set_lm_head")
    enc.vocab = cfg.vocab_size
    enc.max_pos = cfg.max_pos
    return enc


def _snapshot(path, seed):
    """a tiny Llama snapshot (config.json and model.safetensors, vocabulary 256, two layers) of torch seed ``seed``,
    for the DecoderAttention entry points"""
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(vocab_size=256, hidden_size=256, intermediate_size=384, num_hidden_layers=2,
                      num_attention_heads=2, num_key_value_heads=1, head_dim=128, max_position_embeddings=512,
                      rope_theta=10000.0, tie_word_embeddings=False, initializer_range=0.2)
    torch.manual_seed(seed)
    LlamaForCausalLM(cfg).eval().save_pretrained(str(path), safe_serialization=True)
    return str(path)


@pytest.fixture(scope="module")
def snapshots(tmp_path_factory):
    root = tmp_path_factory.mktemp("assisted")
    return [_snapshot(root / f"s{seed}", seed) for seed in (0, 1)]


def _sampling(do_sample=False, temp=1.0, k=50, p=1.0, penalty=1.0):
    L = _lib()
    return L.SamplingC(int(do_sample), temp, p, penalty, k, 0, (C.c_int32 * L.MAX_EOS)())


GREEDY = _sampling(penalty=1.1)
SAMPLED = _sampling(True, 0.7, 50, 0.9, 1.1)


def _plain(enc, ids, s, seed, max_new):
    L = _lib()
    prompt = np.ascontiguousarray(ids, dtype=np.int32)
    out = np.zeros(max_new, dtype=np.int32)
    logits = np.full((max_new, enc.vocab), np.nan, dtype=np.float32)
    n = C.c_int32(0)
    rc = L.lib().rmu_decoder_generate(enc._h, prompt.ctypes.data, len(prompt), C.byref(s), seed, max_new,
                                      out.ctypes.data, C.byref(n), logits.ctypes.data, L.stream_ptr())
    assert rc == 0, L.lib().rmu_last_error()
    return out[:n.value].tolist(), logits


def _assisted(enc, draft, ids, s, seed, max_new, k, schedule=CONSTANT):
    """rmu_decoder_generate_assisted -> (rc, tokens, logits, passes, drafted, kept)"""
    L = _lib()
    prompt = np.ascontiguousarray(ids, dtype=np.int32)
    out = np.zeros(max_new, dtype=np.int32)
    logits = np.full((max_new, enc.vocab), np.nan, dtype=np.float32)
    n, passes, drafted, kept = C.c_int32(0), C.c_int32(-1), C.c_int32(-1), C.c_int32(-1)
    rc = L.lib().rmu_decoder_generate_assisted(enc._h, draft._h if draft is not None else None, prompt.ctypes.data,
                                               len(prompt), C.byref(s), seed, max_new, k, schedule, out.ctypes.data,
                                               C.byref(n), logits.ctypes.data, C.byref(passes), C.byref(drafted),
                                               C.byref(kept), L.stream_ptr())
    return rc, out[:n.value].tolist(), logits, passes.value, drafted.value, kept.value


def _same(a, b):
    """tokens and logits bit for bit; the rows after the last token untouched (NaN) in both"""
    assert a[0] == b[0]
    assert np.array_equal(a[1].view(np.int32), b[1].view(np.int32))


def _check(enc, draft, ids, s, seed, max_new, k, schedule=CONSTANT):
    want = _plain(enc, ids, s, seed, max_new)
    rc, toks, logits, passes, drafted, kept = _assisted(enc, draft, ids, s, seed, max_new, k, schedule)
    assert rc == 0, _lib().lib().rmu_last_error()
    _same((toks, logits), want)
    return passes, drafted, kept


def _cap_passes(T, max_new, k0, max_pos, draft_max_pos):
    """the passes after the prefill when every draft is kept: each pass keeps k + 1 tokens, k capped by
    max_new_tokens, max_pos and the draft's max_pos"""
    n, passes = 1, 0
    while n < max_new and T + n < max_pos:
        p = T + n - 1
        k = max(0, min(k0, 15, max_new - 1 - n, max_pos - 1 - T - n, draft_max_pos - p))
        n, passes = n + k + 1, passes + 1
    return passes


def _prompt(vocab, T, seed=1):
    return np.random.default_rng(seed).integers(0, vocab, T).tolist()


@pytest.mark.parametrize("weights", ["split", "nf4"])
@pytest.mark.parametrize("sampled", [False, True])
def test_same_weights_draft_keeps_every_draft(weights, sampled):
    """a second handle of the target's own weights computes the target's bits in its catch-up rows and its chain:
    every draft is kept, and the passes are those the caps give"""
    enc, draft = _handle(TARGET, weights), _handle(TARGET, weights)
    s = SAMPLED if sampled else GREEDY
    ids = _prompt(enc.vocab, 13)
    for k in (1, 3, 7, 15, 20):
        passes, drafted, kept = _check(enc, draft, ids, s, 5, 40, k)
        assert kept == drafted > 0, (k, drafted, kept)
        assert passes == _cap_passes(len(ids), 40, k, enc.max_pos, draft.max_pos), (k, passes)


@pytest.mark.parametrize("schedule", [CONSTANT, HEURISTIC])
@pytest.mark.parametrize("draft_name", ["synthetic:tiny-llama:7", "synthetic:tiny-llama-draft:2"])
def test_unrelated_draft_equals_plain(draft_name, schedule):
    enc, draft = _handle(TARGET), _handle(draft_name)
    ids = _prompt(enc.vocab, 21, seed=3)
    for s in (GREEDY, SAMPLED):
        for k in (1, 4, 15):
            passes, drafted, kept = _check(enc, draft, ids, s, 9, 30, k, schedule)
            assert 0 <= kept <= drafted


def test_heuristic_schedule_grows_with_a_same_weights_draft():
    """k starts at 1 and grows by 2 per fully kept pass: fewer passes than the constant schedule at k = 1"""
    enc, draft = _handle(TARGET), _handle(TARGET)
    ids = _prompt(enc.vocab, 9)
    const, _, _ = _check(enc, draft, ids, GREEDY, 0, 60, 1, CONSTANT)
    heur, drafted, kept = _check(enc, draft, ids, GREEDY, 0, 60, 1, HEURISTIC)
    assert kept == drafted and heur < const


def test_num_tokens_zero_runs_plain_steps():
    enc, draft = _handle(TARGET), _handle("synthetic:tiny-llama:4")
    passes, drafted, kept = _check(enc, draft, _prompt(enc.vocab, 6), GREEDY, 0, 12, 0)
    assert (passes, drafted, kept) == (11, 0, 0)


@pytest.mark.parametrize("pair", [("split", "nf4"), ("nf4", "split")])
def test_mixed_weights(pair):
    """split target with an NF4 draft and the reverse, on tiny-llama and tiny-qwen3"""
    for name in (TARGET, "synthetic:tiny-qwen3:0"):
        enc, draft = _handle(name, pair[0]), _handle(name, pair[1])
        ids = _prompt(enc.vocab, 17, seed=2)
        for s in (GREEDY, SAMPLED):
            _check(enc, draft, ids, s, 3, 24, 5)


def test_qwen3_32b_layers_with_a_qwen3_06b_draft():
    """two NF4 layers of the Qwen3-32B shape with two layers of the Qwen3-0.6B shape, NF4 and split"""
    enc = _handle("synthetic:qwen3-32b:0", "nf4", layers=2)
    ids = _prompt(enc.vocab, 40, seed=4)
    for weights in ("nf4", "split"):
        draft = _handle("synthetic:qwen3-0.6b:1", weights, layers=2)
        for s in (GREEDY, SAMPLED):
            _check(enc, draft, ids, s, 11, 12, 4)
        del draft


def test_edges():
    """one and two new tokens, a prompt at max_pos - 2, and a draft whose max_pos is below the target's (the draft
    stops drafting once a draft position would reach it)"""
    enc, draft = _handle(TARGET, max_pos=96), _handle(TARGET, max_pos=96)
    ids = _prompt(enc.vocab, 30)
    for s in (GREEDY, SAMPLED):
        for max_new in (1, 2):
            passes, drafted, kept = _check(enc, draft, ids, s, 1, max_new, 7)
            assert passes == max_new - 1 and drafted == 0
        near = _prompt(enc.vocab, 94, seed=5)
        passes, _, _ = _check(enc, draft, near, s, 1, 10, 7)
        assert passes == 1
    short = _handle(TARGET, max_pos=40)
    for s in (GREEDY, SAMPLED):
        passes, drafted, kept = _check(enc, short, ids, s, 2, 30, 7)
        assert kept == drafted and passes == _cap_passes(len(ids), 30, 7, 96, 40)
        # a prompt past the draft's max_pos: no drafting at all
        passes, drafted, _ = _check(enc, short, _prompt(enc.vocab, 50), s, 2, 8, 7)
        assert drafted == 0 and passes == 7


def test_overflowing_draft_never_fails_the_call():
    """a draft whose activations leave the fp16 range (projections ~600) raises its range flag in every pass: each
    pass clears it and proposes nothing, so the call succeeds with the plain tokens in plain steps, and the draft
    serves the next call the same way; its own generate still reports its own range error"""
    enc = _handle(TARGET)
    hot = _handle("synthetic:tiny-llama-draft:5:30000")
    ids = _prompt(enc.vocab, 11)
    for s in (GREEDY, SAMPLED, GREEDY):
        passes, drafted, kept = _check(enc, hot, ids, s, 4, 16, 6)
        assert (passes, drafted, kept) == (15, 0, 0)
    L = _lib()
    prompt = np.ascontiguousarray(ids, dtype=np.int32)
    out = np.zeros(4, dtype=np.int32)
    n = C.c_int32(0)
    assert L.lib().rmu_decoder_generate(hot._h, prompt.ctypes.data, len(prompt), C.byref(GREEDY), 0, 4,
                                        out.ctypes.data, C.byref(n), None, L.stream_ptr()) == -4


def _unloaded_nf4(name):
    """an NF4 handle of ``name`` from rmu_decoder_create_nf4 with no layer loaded, and an LM head"""
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import SyntheticDecoderLayers, decoder_config
    L = _lib()
    cfg = replace(decoder_config(name), vocab_size=1024)
    g = SyntheticDecoderLayers(cfg, seed=0).globals()
    enc = BertEncoder.__new__(BertEncoder)
    enc.torch, enc.cfg, enc.device, enc._h = torch, cfg, torch.device("cuda", 0), C.c_void_p()
    cos, sin = (np.ascontiguousarray(t, np.float32) for t in cfg.rope_tables())
    cc, qx = L.bert_config_c(cfg), L.Qwen3ExtC(cfg.kv_heads, 128, cfg.max_pos, 64, 0, -1)
    L.check(L.lib().rmu_decoder_create_nf4(C.byref(cc), C.byref(qx), 0, g["embed_tokens.weight"].ctypes.data,
                                           g["norm.weight"].ctypes.data, cos.ctypes.data, sin.ctypes.data,
                                           C.byref(enc._h)), "rmu_decoder_create_nf4")
    lm = np.ascontiguousarray(0.02 * np.random.default_rng(1).standard_normal((cfg.vocab_size, cfg.hidden)),
                              dtype=np.float32)
    L.check(L.lib().rmu_decoder_set_lm_head(enc._h, lm.ctypes.data), "rmu_decoder_set_lm_head")
    return enc


def test_refusals_on_live_handles():
    """a vocabulary mismatch (naming both sizes), the target as its own draft, a draft without an LM head, an NF4
    draft with a layer missing, num_tokens < 0 and an unknown schedule"""
    L = _lib()
    enc = _handle(TARGET)
    ids = _prompt(enc.vocab, 5)
    rc, *_ = _assisted(enc, _handle("synthetic:qwen3-0.6b:0", "nf4", layers=1), ids, GREEDY, 0, 4, 3)
    msg = L.lib().rmu_last_error().decode()
    assert rc == -1 and "151936" in msg and "1024" in msg
    rc, *_ = _assisted(enc, enc, ids, GREEDY, 0, 4, 3)
    assert rc == -1 and "another handle" in L.lib().rmu_last_error().decode()
    rc, *_ = _assisted(enc, _handle("synthetic:tiny-llama:2", lm_head=False), ids, GREEDY, 0, 4, 3)
    assert rc == -1 and "LM head" in L.lib().rmu_last_error().decode()
    rc, *_ = _assisted(enc, _unloaded_nf4("synthetic:tiny-llama-draft:0"), ids, GREEDY, 0, 4, 3)
    assert rc == -1 and "layer 0 of 1 is not loaded" in L.lib().rmu_last_error().decode()
    draft = _handle("synthetic:tiny-llama:1")
    rc, *_ = _assisted(enc, draft, ids, GREEDY, 0, 4, -1)
    assert rc == -1
    rc, *_ = _assisted(enc, draft, ids, GREEDY, 0, 4, 2, schedule=7)
    assert rc == -1 and "schedule" in L.lib().rmu_last_error().decode()
    # the refused calls left both handles working
    _check(enc, draft, ids, GREEDY, 0, 8, 3)


def test_concurrent_session_and_assisted_call(snapshots):
    """an assisted call and a session generate on the same target from two threads: both equal their solo runs"""
    from ragmeup_b200 import provenance
    a = provenance.DecoderAttention(snapshots[0])
    b = provenance.DecoderAttention(snapshots[1])
    ids1, ids2 = _prompt(256, 12, seed=6), _prompt(256, 8, seed=7)
    kw = dict(do_sample=True, temperature=0.7, top_k=50, top_p=0.9, repetition_penalty=1.1)
    want1 = a.generate(ids1, 30, seed=1, **kw)
    want2 = a.generate(ids2, 30, seed=2, **kw)
    got = {}
    t1 = threading.Thread(target=lambda: got.update(x=a.generate(ids1, 30, seed=1, assistant=b, num_assistant_tokens=5,
                                                                 **kw)), daemon=True)
    t2 = threading.Thread(target=lambda: got.update(y=a.generate(ids2, 30, seed=2, **kw)), daemon=True)
    t1.start(); t2.start()
    t1.join(120); t2.join(120)
    assert not t1.is_alive() and not t2.is_alive()
    assert got["x"] == want1 and got["y"] == want2


def test_swapped_roles_do_not_deadlock(snapshots):
    from ragmeup_b200 import provenance
    a = provenance.DecoderAttention(snapshots[0])
    b = provenance.DecoderAttention(snapshots[1])
    ids = _prompt(256, 10, seed=8)
    want_a, want_b = a.generate(ids, 40), b.generate(ids, 40)
    got = {}
    t1 = threading.Thread(target=lambda: got.update(a=a.generate(ids, 40, assistant=b, num_assistant_tokens=4)),
                          daemon=True)
    t2 = threading.Thread(target=lambda: got.update(b=b.generate(ids, 40, assistant=a, num_assistant_tokens=4)),
                          daemon=True)
    t1.start(); t2.start()
    t1.join(120); t2.join(120)
    assert not t1.is_alive() and not t2.is_alive()
    assert got["a"] == want_a and got["b"] == want_b


def test_decoder_attention_and_pipeline(tmp_path, monkeypatch, snapshots):
    """DecoderAttention.generate(assistant=...) equals plain generate; HuggingFacePipeline with assistant_model (the
    transformers model of a second copy of the chat snapshot, another decoder handle) and with RMU_ASSISTANT_MODEL
    naming that copy return the plain text"""
    from transformers import AutoModelForCausalLM, AutoTokenizer, pipeline
    from ragmeup_b200 import llms, provenance
    a = provenance.DecoderAttention(snapshots[0])
    d = provenance.DecoderAttention(snapshots[1])
    ids = _prompt(256, 15, seed=9)
    for kw in (dict(), dict(do_sample=True, temperature=0.7, top_k=30, top_p=0.9, repetition_penalty=1.1, seed=4)):
        want = a.generate(ids, 20, **kw)
        for k, sched in ((3, "constant"), (20, "heuristic"), (2, "heuristic_transient")):
            assert a.generate(ids, 20, assistant=d, num_assistant_tokens=k, num_assistant_tokens_schedule=sched,
                              **kw) == want
    with pytest.raises(ValueError, match="prompt_lookup_num_tokens.*assistant"):
        a.generate(ids, 4, assistant=d, prompt_lookup_num_tokens=3)
    target_dir, draft_dir = tmp_path / "target", tmp_path / "draft"
    mg.save_chat_snapshot(str(target_dir))
    mg.save_chat_snapshot(str(draft_dir))
    model = AutoModelForCausalLM.from_pretrained(str(target_dir)).eval()
    tok = AutoTokenizer.from_pretrained(str(target_dir))
    prompt = "w5 w6 w7 w8 w9 w5 w6 w7 w8 w9 w5 w6 " + mg.ASSISTANT
    monkeypatch.delenv(llms.PROMPT_LOOKUP_ENV, raising=False)
    monkeypatch.delenv(llms.ASSISTANT_ENV, raising=False)
    draft_model = AutoModelForCausalLM.from_pretrained(str(draft_dir)).eval()

    for sample in (dict(do_sample=False), dict(do_sample=True, temperature=0.6, top_p=0.9)):
        pipe = pipeline(model=model, tokenizer=tok, task="text-generation", repetition_penalty=1.1,
                        return_full_text=True, max_new_tokens=16, **sample)
        torch.manual_seed(0)
        want = llms.HuggingFacePipeline(pipeline=pipe).invoke(prompt)
        pipe_a = pipeline(model=model, tokenizer=tok, task="text-generation", repetition_penalty=1.1,
                          return_full_text=True, max_new_tokens=16, assistant_model=draft_model, **sample)
        torch.manual_seed(0)
        assert llms.HuggingFacePipeline(pipeline=pipe_a).invoke(prompt) == want
        monkeypatch.setenv(llms.ASSISTANT_ENV, str(draft_dir))
        torch.manual_seed(0)
        assert llms.HuggingFacePipeline(pipeline=pipe).invoke(prompt) == want
        monkeypatch.delenv(llms.ASSISTANT_ENV)
