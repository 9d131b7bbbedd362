"""70B-class decoders on the GPU: the wide RMSNorm against float64; NF4 handles built layer by layer
(rmu_decoder_create_nf4 / rmu_decoder_load_layer_nf4) against split upload + rmu_decoder_quantize_nf4, bit for bit;
the refusals of a handle whose layers are not all loaded; two layers of the Llama-3.1-70B and Qwen3-32B shapes against
the float64 forward on oracle/nf4_ref.py's dequantised weights, with batched, session and prompt-lookup generation
each equal to single generation; and the release of the reference's transformers copy of the model."""
from __future__ import annotations

import ctypes as C
import gc
from dataclasses import replace

import numpy as np
import pytest
import torch

import make_golden_generate as mg
from oracle import decoder_attention_ref as da
from oracle import nf4_ref as nf4
from test_decode_batch_gpu import _batch, _handle, _prompts, _sampling, _single
from test_decode_session_gpu import Tracker

pytestmark = pytest.mark.gpu

PROJ = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


@pytest.fixture(autouse=True)
def _release_torch_cache():
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _lib():
    from ragmeup_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------------------ wide norm
@pytest.mark.parametrize("H", [4224, 5120, 6144, 8192])
def test_wide_rmsnorm_against_float64(H):
    """the 256-thread form above 4096 (4224: a row that ends inside a thread block's last column pass)"""
    L = _lib()
    g = torch.Generator(device="cuda").manual_seed(H)
    T = 300
    x = torch.randn(T, H, device="cuda", generator=g) * 3
    x[1] *= 1e-3
    w = 1 + 0.2 * torch.randn(H, device="cuda", generator=g)
    hi = torch.full((T, H), float("nan"), dtype=torch.float16, device="cuda")
    lo = torch.full_like(hi, float("nan"))
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(L.lib().rmu_debug_rmsnorm(x.data_ptr(), T, H, w.data_ptr(), 1e-5, hi.data_ptr(), lo.data_ptr(),
                                      flag.data_ptr(), L.stream_ptr()), "rmsnorm")
    torch.cuda.synchronize()
    X = x.double()
    want = w.double() * (X * torch.rsqrt(X.pow(2).mean(-1, keepdim=True) + 1e-5))
    err = float(((hi.double() + lo.double() - want).abs() / want.abs().amax(1, keepdim=True)).max())
    assert err <= 2e-6 and int(flag.item()) == 0, err
    # a large gain on the last column: y = 2000 x / rms(x) stays below 10 000 on every row of N(0, 9) values, and only
    # row 7, whose last value dominates it (y = 2000 sqrt(H) > 65 504), leaves the fp16 range
    w_big = w.clone()
    w_big[H - 1] = 2000.0
    L.check(L.lib().rmu_debug_rmsnorm(x.data_ptr(), T, H, w_big.data_ptr(), 1e-5, hi.data_ptr(), lo.data_ptr(),
                                      flag.data_ptr(), L.stream_ptr()), "rmsnorm")
    torch.cuda.synchronize()
    assert int(flag.item()) == 0
    x[7, H - 1] = 1e9
    L.check(L.lib().rmu_debug_rmsnorm(x.data_ptr(), T, H, w_big.data_ptr(), 1e-5, hi.data_ptr(), lo.data_ptr(),
                                      flag.data_ptr(), L.stream_ptr()), "rmsnorm")
    torch.cuda.synchronize()
    assert int(flag.item()) == 1
    y = hi.double() + lo.double()
    assert not torch.isfinite(y[7]).all() and torch.isfinite(torch.cat([y[:7], y[8:]])).all()
    assert L.lib().rmu_debug_rmsnorm(x.data_ptr(), T, 8320, w.data_ptr(), 1e-5, hi.data_ptr(), lo.data_ptr(), None,
                                     None) == -3


# ---------------------------------------------------------------------------------------------- layered handles
def _layered(cfg, w, lm=None, on_layer=None):
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import DictDecoderLayers
    enc = BertEncoder.nf4_decoder(DictDecoderLayers(cfg, w), on_layer=on_layer)
    if lm is not None:
        L = _lib()
        enc._check(L.lib().rmu_decoder_set_lm_head(enc._h, np.ascontiguousarray(lm).ctypes.data), "set_lm_head")
    return enc


def _spans(enc, ids, spans):
    L = _lib()
    d_ids = torch.as_tensor(np.asarray(ids, np.int32), device="cuda")
    d_sp = torch.as_tensor(np.asarray(spans, np.int32).reshape(-1, 2), device="cuda")
    out = torch.empty((len(spans), len(spans)), dtype=torch.float64, device="cuda")
    enc._check(L.lib().rmu_decoder_attention_spans(enc._h, d_ids.data_ptr(), len(ids), d_sp.data_ptr(), len(spans),
                                                   out.data_ptr(), L.stream_ptr()), "spans")
    return out.cpu().numpy()


def _eight_b_two_layers():
    from ragmeup_b200.weights import DECODER_PRESETS, synthetic_llama_weights
    cfg = replace(DECODER_PRESETS["llama-3.1-8b"], layers=2, vocab_size=2048, max_pos=4096)
    lm = (np.random.default_rng(4).standard_normal((cfg.vocab_size, cfg.hidden)) * 0.05).astype(np.float32)
    return cfg, synthetic_llama_weights(cfg, seed=4), lm


@pytest.mark.parametrize("kind", ["llama", "qwen3", "llama-8b"])
def test_layered_handle_is_the_converted_handle(kind):
    """the same codes as split upload + rmu_decoder_quantize_nf4, seen through every output: generate's tokens and
    logits (greedy and sampled, prompts of 1 and several tokens) and span_mass, bit for bit"""
    cfg, w, lm = _eight_b_two_layers() if kind == "llama-8b" else mg.model(kind)
    qk = kind == "qwen3"
    *_, ref = _handle("qwen3" if qk else "llama", "nf4", cfg_w_lm=(cfg, w, lm))
    enc = _layered(cfg, w, lm)
    V = cfg.vocab_size
    rng = np.random.default_rng(7)
    for T in (1, 37, 300):
        ids = rng.integers(0, V, T).tolist()
        for s, seed in ((_sampling(), 0), (_sampling(True, 0.8, 40, 0.9, 1.1), 1234)):
            a, la = _single(ref, V, ids, s, seed, 10)
            b, lb = _single(enc, V, ids, s, seed, 10)
            assert a == b and np.array_equal(la.view(np.int32), lb.view(np.int32)), (T, seed)
    ids = rng.integers(0, V, 400).tolist()
    spans = [(0, 400), (10, 120), (120, 300), (300, 399)]
    assert np.array_equal(_spans(ref, ids, spans).view(np.int64), _spans(enc, ids, spans).view(np.int64))


def test_incomplete_handle_and_load_refusals():
    """layers load in order; until the last is in, every forward, span, generate and session entry refuses naming the
    missing layer; a weight outside the split planes' range is refused naming its layer and projection, and the layer
    then loads"""
    from ragmeup_b200.weights import DictDecoderLayers
    L = _lib()
    l = L.lib()
    cfg, w, lm = mg.model("llama")
    src = DictDecoderLayers(cfg, w)
    from ragmeup_b200.encoder import BertEncoder
    enc = BertEncoder.__new__(BertEncoder)
    enc.torch, enc.cfg, enc.device, enc._h = torch, cfg, torch.device("cuda", 0), C.c_void_p()
    g = src.globals()
    cos, sin = (np.ascontiguousarray(t, np.float32) for t in cfg.rope_tables())
    cc, qx = L.bert_config_c(cfg), L.Qwen3ExtC(cfg.kv_heads, 128, cfg.max_pos, 64, 0, -1)
    L.check(l.rmu_decoder_create_nf4(C.byref(cc), C.byref(qx), 0, g["embed_tokens.weight"].ctypes.data,
                                     g["norm.weight"].ctypes.data, cos.ctypes.data, sin.ctypes.data, C.byref(enc._h)),
            "create")

    def load(layer, t=None, tensors_of=None):
        """layer `layer` from the tensors of layer `tensors_of` (default: its own), always a full set of 9"""
        own = layer if tensors_of is None else tensors_of
        t = t or src.layer(own)
        arrs = [np.ascontiguousarray(t[n], np.float32) for n, _ in src.layer_names(own)]
        assert len(arrs) == 9
        return l.rmu_decoder_load_layer_nf4(enc._h, layer, (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs]),
                                            None)
    outside = b"outside the model's 3 layers"
    assert load(3, tensors_of=2) == -1 and outside in l.rmu_last_error()
    assert load(-1, tensors_of=0) == -1 and outside in l.rmu_last_error()
    assert load(0) == 0
    assert load(2) == -1 and b"expected layer 1 of 3, got 2" in l.rmu_last_error()
    assert load(0) == -1
    enc._check(l.rmu_decoder_set_lm_head(enc._h, np.ascontiguousarray(lm).ctypes.data), "set_lm_head")
    s = _sampling()
    prompt = np.arange(5, dtype=np.int32)
    out, n = np.zeros(4, np.int32), C.c_int32(0)
    missing = b"layer 1 of 3 is not loaded"
    assert l.rmu_decoder_generate(enc._h, prompt.ctypes.data, 5, C.byref(s), 0, 4, out.ctypes.data, C.byref(n), None,
                                  None) == -1 and missing in l.rmu_last_error()
    assert l.rmu_decoder_generate_lookup(enc._h, prompt.ctypes.data, 5, C.byref(s), 0, 4, 3, 2, out.ctypes.data,
                                         C.byref(n), None, None, None) == -1 and missing in l.rmu_last_error()
    rc, *_ = _batch(enc, cfg.vocab_size, [[1, 2], [1, 3]], s, [0, 1], 4)
    assert rc == -1 and missing in l.rmu_last_error()
    with pytest.raises(L.RmuError, match="layer 1 of 3 is not loaded"):
        _spans(enc, [1, 2, 3], [(0, 3)])
    with pytest.raises(L.RmuError, match="layer 1 of 3 is not loaded"):
        enc.hidden_tokens(prompt, None, np.array([0, 5], np.int32), 5)
    sess = C.c_void_p()
    assert l.rmu_decoder_session_create(enc._h, C.byref(sess)) == -1 and missing in l.rmu_last_error()
    bad = dict(src.layer(1))
    bad["layers.1.mlp.gate_proj.weight"] = bad["layers.1.mlp.gate_proj.weight"].copy()
    bad["layers.1.mlp.gate_proj.weight"][3, 5] = 7e4
    assert load(1, bad) == -3
    assert b"layer 1 gate_proj weight [" in l.rmu_last_error() and b"65520" in l.rmu_last_error()
    assert load(1) == 0 and load(2) == 0
    # every layer is in: one past the last, and any repeat, are refused and change nothing
    assert load(3, tensors_of=2) == -1 and outside in l.rmu_last_error()
    assert load(2) == -1 and b"expected layer 3 of 3, got 2" in l.rmu_last_error()
    ref = _layered(cfg, w, lm)
    a, la = _single(ref, cfg.vocab_size, prompt.tolist(), s, 0, 6)
    b, lb = _single(enc, cfg.vocab_size, prompt.tolist(), s, 0, 6)
    assert a == b and np.array_equal(la.view(np.int32), lb.view(np.int32))


# ---------------------------------------------------------------------------------------------- wide shapes
def _quantize_dequantize(v):
    """v's NF4 dequantised weight through the device quantiser and dequantiser, both bit for bit nf4_ref.quantize /
    nf4_ref.dequantize (test_nf4_gpu); the first rows are also checked against nf4_ref.nf4_weight itself here"""
    L = _lib()
    hi = v.to(torch.float16).reshape(-1)
    n = hi.numel()
    codes = torch.empty(n // 2, dtype=torch.uint8, device="cuda")
    absmax = torch.empty(n // 64, dtype=torch.float32, device="cuda")
    L.check(L.lib().rmu_debug_nf4_quantize(hi.data_ptr(), n, codes.data_ptr(), absmax.data_ptr(), L.stream_ptr()), "q")
    L.check(L.lib().rmu_debug_nf4_dequantize(codes.data_ptr(), absmax.data_ptr(), n, hi.data_ptr(), L.stream_ptr()), "d")
    d = hi.reshape(v.shape).float()
    head = v[:64].cpu().numpy()
    assert np.array_equal(d[:64].cpu().numpy(), nf4.nf4_weight(head))
    return d


def _wide(preset):
    """two layers of the preset's shape with a 1 024-token vocabulary: weights drawn on the device (norms 1 + N(0, 0.1),
    embeddings N(0, 0.06), projections N(0, 0.02) as transformers initialises them), as host fp32 for the handle and as CUDA fp32 for the oracle, whose
    projections are the NF4 dequantised ones"""
    from ragmeup_b200.weights import decoder_config, decoder_weight_names
    cfg = replace(decoder_config("synthetic:" + preset), layers=2, vocab_size=1024, max_pos=4096)
    g = torch.Generator(device="cuda").manual_seed(2)
    w, W = {}, {}
    for name, shape in decoder_weight_names(cfg):
        a = torch.randn(shape, generator=g, device="cuda")
        norm = name.endswith("norm.weight") or name.endswith("layernorm.weight")
        a = 1 + 0.1 * a if norm else (0.06 if name == "embed_tokens.weight" else 0.02) * a
        w[name] = a.cpu().numpy()
        W[name] = _quantize_dequantize(a) if any(name.endswith(p + ".weight") for p in PROJ) else a
        del a
    lm = (torch.randn(cfg.vocab_size, cfg.hidden, generator=g, device="cuda") * 0.3).cpu().numpy()
    return cfg, w, W, lm, preset.startswith("qwen3")


def _oracle_logits(W, lm64, cfg, ids, qk):
    h = da.hidden(W, cfg, ids, torch.float64, qk)[-1]
    return (lm64 @ h).cpu().numpy()


@pytest.mark.parametrize("preset", ["llama-3.1-70b", "qwen3-32b"])
def test_wide_shapes_against_float64(preset):
    """two layers of the 70B-class shapes (hidden 8192 and 5120, 8 query heads per kv head, down projection K = 28 672
    and 25 600): the prefill's logits and greedy decode steps against the float64 forward on the dequantised NF4
    weights, within the NF4 whole-handle tolerance of the decode steps (1e-4 of the largest logit; the tiny shapes'
    2e-5 bound on the prefill does not carry over to these K).  At the Qwen3-32B shape also: rmu_decoder_generate_batch, a
    two-request decode session and prompt lookup each equal single generation bit for bit, and span_mass against the
    oracle."""
    L = _lib()
    cfg, w, W, lm, qk = _wide(preset)
    enc = _layered(cfg, w, lm)
    del w
    lm64 = torch.as_tensor(lm, device="cuda", dtype=torch.float64)
    V = cfg.vocab_size
    rng = np.random.default_rng(3)
    for T in (1, 24, 200):
        ids = rng.integers(0, V, T).tolist()
        N = 4
        toks, logits = _single(enc, V, ids, _sampling(), 0, N)
        assert len(toks) == N
        refs = [_oracle_logits(W, lm64, cfg, ids + toks[:t], qk) for t in range(N)]
        err = [float(np.abs(logits[t] - refs[t]).max() / np.abs(refs[t]).max()) for t in range(N)]
        print(f"\n{preset} T={T}: max |logit error| / max |logit|, prefill then steps: "
              + " ".join(f"{e:.2e}" for e in err))
        assert max(err) <= 1e-4, (T, err)
        for t, ref in enumerate(refs):
            top2 = np.sort(ref)[-2:]
            if top2[1] - top2[0] <= 1e-4 * np.abs(ref).max():
                break
            assert toks[t] == int(np.argmax(ref)), (T, t)
    if not qk:
        return
    # batched, session and prompt-lookup generation against single generation, bit for bit
    s = _sampling(True, 0.7, 50, 0.9, 1.1)
    prompts = _prompts(V, 3, 40, 8, [1, 17, 60])
    seeds = [5, 6, 7]
    rc, out, n, lg = _batch(enc, V, prompts, s, seeds, 8)
    assert rc == 0, L.lib().rmu_last_error()
    for b, p in enumerate(prompts):
        toks, lgs = _single(enc, V, p, s, seeds[b], 8)
        assert out[b, :n[b]].tolist() == toks and np.array_equal(lg[b, :n[b]].view(np.int32), lgs.view(np.int32))
    t = Tracker(enc, V)
    t.add([("a", prompts[1], s, 11, 8)])
    t.step()
    t.add([("b", prompts[2], _sampling(), 12, 8)])
    t.run()
    t.check(enc)
    ids = (list(range(30, 50)) * 4)[:70]
    greedy = _sampling()
    want, lw = _single(enc, V, ids, greedy, 0, 12)
    out = np.zeros(12, np.int32)
    got_l = np.zeros((12, V), np.float32)
    nn, passes = C.c_int32(0), C.c_int32(0)
    prompt = np.ascontiguousarray(ids, np.int32)
    enc._check(L.lib().rmu_decoder_generate_lookup(enc._h, prompt.ctypes.data, len(ids), C.byref(greedy), 0, 12, 5, 2,
                                                   out.ctypes.data, C.byref(nn), got_l.ctypes.data, C.byref(passes),
                                                   L.stream_ptr()), "lookup")
    assert out[:nn.value].tolist() == want and np.array_equal(got_l[:nn.value].view(np.int32), lw.view(np.int32))
    ids = rng.integers(0, V, 120).tolist()
    spans = [(0, 120), (5, 40), (40, 119)]
    got = _spans(enc, ids, spans)
    A = da.last_attention(W, cfg, ids, qk_norm=True)
    want = torch.stack([torch.stack([A[:, a0:a1, b0:b1].sum() for b0, b1 in spans]) for a0, a1 in spans]).cpu().numpy()
    size = np.array([e - s0 for s0, e in spans], np.float64)
    assert (np.abs(got - want) <= 1e-4 * cfg.heads * size[:, None]).all()


# ---------------------------------------------------------------------------------------------- release
def test_release_of_the_transformers_copy(tmp_path, monkeypatch):
    """a transformers causal LM on CUDA and free memory reported too low for the decoder beside it: its parameters are
    freed, torch's allocator hands the memory back, and HuggingFacePipeline still generates what the CPU pipeline
    generates"""
    from transformers import AutoModelForCausalLM, AutoTokenizer, pipeline
    from ragmeup_b200 import provenance
    from ragmeup_b200.llms import HuggingFacePipeline
    monkeypatch.setattr(provenance, "_DECODERS", {})
    monkeypatch.delenv("RMU_DECODER_WEIGHTS", raising=False)
    mg.save_chat_snapshot(str(tmp_path))
    tok = AutoTokenizer.from_pretrained(str(tmp_path))
    kw = dict(task="text-generation", temperature=0.6, repetition_penalty=1.1, return_full_text=True, max_new_tokens=16,
              do_sample=False)
    prompt = "w5 w6 w7 w8 w9 w10 w11 " + mg.ASSISTANT
    with torch.no_grad():
        want = pipeline(model=AutoModelForCausalLM.from_pretrained(str(tmp_path)).eval(), tokenizer=tok, **kw)(
            prompt)[0]["generated_text"]
    model = AutoModelForCausalLM.from_pretrained(str(tmp_path)).cuda().eval()
    pipe = pipeline(model=model, tokenizer=tok, **kw)
    n_bytes = sum(p.numel() * p.element_size() for p in model.parameters())
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    real = torch.cuda.mem_get_info
    calls = []

    def low_once(device=None):
        calls.append(device)
        free, total = real(device)
        return (1 << 20, total) if len(calls) == 1 else (free, total)
    monkeypatch.setattr(torch.cuda, "mem_get_info", low_once)
    got = HuggingFacePipeline(pipeline=pipe).invoke(prompt)
    assert got == want
    assert all(p.numel() == 0 and not p.is_cuda for p in model.parameters())
    assert before - torch.cuda.memory_allocated() >= n_bytes
    assert model.name_or_path == str(tmp_path) and model.generation_config is not None and model.config is not None
    # a decoder that fits leaves the model alone
    model2 = AutoModelForCausalLM.from_pretrained(str(tmp_path)).cuda().eval()
    monkeypatch.setattr(provenance, "_DECODERS", {})
    assert provenance.release_model_if_needed(model2, 1 << 20, torch.cuda.current_device()) == 0
    assert all(p.is_cuda and p.numel() > 0 for p in model2.parameters())
