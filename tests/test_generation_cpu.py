"""Generation without a GPU: the oracle's processors against transformers' logits processors, its greedy generation
against transformers' LlamaForCausalLM / Qwen3ForCausalLM in float64, the settings HuggingFacePipeline resolves and
refuses, and the C entry points' refusals."""
from __future__ import annotations

import ctypes as C
from dataclasses import replace

import os

import numpy as np
import pytest
import torch

import make_golden_generate as mg

from oracle import generation_ref as gref
from ragmeup_b200.weights import DECODER_PRESETS, PRESETS, synthetic_llama_weights, synthetic_qwen3_weights


def _logits(seed, V=300):
    rng = np.random.default_rng(seed)
    x = np.round(rng.standard_normal(V) * 4, 1)                 # rounding plants ties
    x[[3, 70, 250]] = x.max()
    return x


@pytest.mark.parametrize("seed", range(6))
def test_processors_match_transformers(seed):
    from transformers import (RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper, TopKLogitsWarper,
                              TopPLogitsWarper)
    x = _logits(seed)
    seen = [3, 5, 9, 9, 120, 299]
    t = torch.tensor(x, dtype=torch.float64)[None]
    ids = torch.tensor(seen)[None]
    assert np.array_equal(RepetitionPenaltyLogitsProcessor(1.3)(ids, t.clone())[0].numpy(),
                          gref.repetition_penalty(x, seen, 1.3))
    assert np.array_equal(TemperatureLogitsWarper(0.7)(ids, t.clone())[0].numpy(), gref.temperature(x, 0.7))
    for k in (1, 5, 40, 256):
        assert np.array_equal(TopKLogitsWarper(k)(ids, t.clone())[0].numpy(), gref.top_k(x, k))
    # torch.sort leaves the order of equal values unspecified: top-p is compared on distinct values
    xd = x + np.arange(x.size) * 1e-9
    td = torch.tensor(xd, dtype=torch.float64)[None]
    for p in (0.3, 0.9, 0.99):
        assert np.array_equal(TopPLogitsWarper(p)(ids, td.clone())[0].numpy(), gref.top_p(xd, p))


@pytest.mark.parametrize("seed", range(4))
def test_sampler_rule_agrees_with_processors(seed):
    """without more than 256 survivors, the sampler's candidates and top-p are transformers' top-k then top-p"""
    x = _logits(seed) + np.arange(300) * 1e-9
    for k, p in ((5, 1.0), (40, 0.9), (200, 0.5)):
        want = np.isfinite(gref.top_p(gref.top_k(x, k), p))
        c = gref.kept(x, gref.candidates(x, k), p)
        got = np.zeros(x.size, bool)
        got[c] = True
        assert np.array_equal(got, want)


def test_philox_uniform():
    # Random123's known-answer vectors for philox4x32_10
    assert gref.philox4x32_10([0, 0, 0, 0], [0, 0]) == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    assert gref.philox4x32_10([0xffffffff] * 4, [0xffffffff] * 2) == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    assert gref.philox4x32_10([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344],
                              [0xa4093822, 0x299f31d0]) == [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]
    assert gref.philox_uniform(0, 0) == (0x6627e8d5 >> 8) / 2 ** 24
    u = [gref.philox_uniform(s, t) for s in (0, 1, 2 ** 40 + 3) for t in (0, 1, 7)]
    assert all(0.0 <= v < 1.0 for v in u) and len(set(u)) == len(u)
    assert gref.philox_uniform(5, 3) == gref.philox_uniform(5, 3)


@pytest.mark.parametrize("kind", ["llama", "qwen3"])
def test_oracle_greedy_matches_transformers(kind):
    if kind == "llama":
        from transformers import LlamaConfig as HC, LlamaForCausalLM as M
        cfg = replace(DECODER_PRESETS["tiny-llama"], layers=2, max_pos=64)
        w = synthetic_llama_weights(cfg, seed=1, scale=4.0)
        rs = cfg.rope_scaling
        hc = HC(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, intermediate_size=cfg.ffn, num_hidden_layers=cfg.layers,
                num_attention_heads=cfg.heads, num_key_value_heads=cfg.kv_heads, head_dim=128,
                max_position_embeddings=cfg.max_pos, rms_norm_eps=cfg.ln_eps, rope_theta=cfg.rope_theta,
                rope_scaling={"rope_type": "llama3", "factor": rs[0], "low_freq_factor": rs[1], "high_freq_factor": rs[2],
                              "original_max_position_embeddings": rs[3], "rope_theta": cfg.rope_theta},
                tie_word_embeddings=False)
    else:
        from transformers import Qwen3Config as HC, Qwen3ForCausalLM as M
        cfg = replace(PRESETS["tiny-qwen3"][0], layers=2, max_pos=64)
        w = synthetic_qwen3_weights(cfg, seed=1, scale=4.0)
        hc = HC(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, intermediate_size=cfg.ffn, num_hidden_layers=cfg.layers,
                num_attention_heads=cfg.heads, num_key_value_heads=cfg.kv_heads, head_dim=128,
                max_position_embeddings=cfg.max_pos, rms_norm_eps=cfg.ln_eps, rope_theta=cfg.rope_theta,
                tie_word_embeddings=False)
    lm = (np.random.default_rng(2).standard_normal((cfg.vocab_size, cfg.hidden)) * 0.5).astype(np.float32)
    model = M(hc).to(torch.float64).eval()
    sd = {"model." + k: torch.tensor(v, dtype=torch.float64) for k, v in w.items()}
    sd["lm_head.weight"] = torch.tensor(lm, dtype=torch.float64)
    model.load_state_dict(sd, strict=False)
    ids = [5, 17, 3, 250, 9, 41]
    with torch.no_grad():
        out = model.generate(torch.tensor([ids]), max_new_tokens=8, do_sample=False, repetition_penalty=1.2,
                             pad_token_id=0, eos_token_id=None)
    want = out[0, len(ids):].tolist()
    assert gref.generate(w, lm, cfg, ids, 8, qk_norm=kind == "qwen3", penalty=1.2) == want


def test_settings_resolution_and_refusals():
    from transformers import GenerationConfig
    from ragmeup_b200.llms import resolve_settings
    gc = GenerationConfig(do_sample=True, temperature=0.6, top_p=0.9, eos_token_id=[128001, 128008, 128009])
    s = resolve_settings(gc, {"max_new_tokens": 7, "repetition_penalty": 1.1}, 10)
    assert s == dict(max_new_tokens=7, do_sample=True, temperature=0.6, top_k=50, top_p=0.9, repetition_penalty=1.1,
                     eos_token_ids=[128001, 128008, 128009])
    assert resolve_settings(GenerationConfig(), {}, 4)["max_new_tokens"] == 16          # max_length 20
    assert gc.temperature == 0.6 and gc.max_new_tokens is None                          # the caller's config is kept
    for kw, field in (({"num_beams": 2}, "num_beams"), ({"num_return_sequences": 2}, "num_return_sequences"),
                      ({"min_p": 0.1}, "min_p"), ({"typical_p": 0.5}, "typical_p"),
                      ({"no_repeat_ngram_size": 3}, "no_repeat_ngram_size"), ({"bad_words_ids": [[1]]}, "bad_words_ids"),
                      ({"sequence_bias": {(1,): 1.0}}, "sequence_bias"), ({"suppress_tokens": [1]}, "suppress_tokens"),
                      ({"forced_bos_token_id": 1}, "forced_bos_token_id"), ({"min_new_tokens": 2}, "min_new_tokens"),
                      ({"min_length": 5}, "min_length"), ({"stop_strings": ["x"]}, "stop_strings"),
                      ({"epsilon_cutoff": 1e-3}, "epsilon_cutoff"), ({"eta_cutoff": 1e-3}, "eta_cutoff"),
                      ({"guidance_scale": 2.0}, "guidance_scale"), ({"do_sample": True, "top_k": 0}, "top_k"),
                      ({"do_sample": True, "top_k": 300}, "top_k"), ({"no_such_setting": 1}, "no_such_setting")):
        with pytest.raises(ValueError, match=field):
            resolve_settings(GenerationConfig(), kw, 4)


def test_c_refusals():
    from ragmeup_b200 import _lib
    L = _lib.lib()
    s = _lib.SamplingC(1, 1.0, 1.0, 1.0, 0, 0, (C.c_int32 * _lib.MAX_EOS)())
    out = np.zeros(4, np.int32)
    n = C.c_int32()
    ids = np.zeros(3, np.int32)
    assert L.rmu_decoder_set_lm_head(None, None) == -1
    assert L.rmu_decoder_generate(None, ids.ctypes.data, 3, C.byref(s), 0, 4, out.ctypes.data, C.byref(n), None,
                                  None) == -1
    x = np.zeros(8, np.float32)
    assert L.rmu_debug_sample(x.ctypes.data, 8, x.ctypes.data, C.byref(s), 0.5, x.ctypes.data, None) == -3   # top_k 0
    s.top_k = 257
    assert L.rmu_debug_sample(x.ctypes.data, 8, x.ctypes.data, C.byref(s), 0.5, x.ctypes.data, None) == -3
    s.top_k, s.temperature = 5, 0.0
    assert L.rmu_debug_sample(x.ctypes.data, 8, x.ctypes.data, C.byref(s), 0.5, x.ctypes.data, None) == -1
    s.temperature, s.n_eos = 1.0, 9
    assert L.rmu_debug_sample(x.ctypes.data, 8, x.ctypes.data, C.byref(s), 0.5, x.ctypes.data, None) == -1
    s.n_eos = 0
    assert L.rmu_debug_sample(x.ctypes.data, 8, x.ctypes.data, C.byref(s), 1.0, x.ctypes.data, None) == -1   # u = 1
    p = x.ctypes.data
    assert L.rmu_debug_attention_decode(p, p, p, 3, 2, 8, 4, p, 4096, p, p, None) == -3
    assert L.rmu_debug_attention_decode(p, p, p, 2, 2, 8, 9, p, 4096, p, p, None) == -1


def test_golden_fixture_matches_oracle(golden_dir):
    z = np.load(os.path.join(golden_dir, "generate.npz"))
    want = mg.compute()
    assert sorted(z.files) == sorted(want)
    for k, v in want.items():
        if k.endswith("_logits"):
            assert np.allclose(z[k], v, rtol=1e-12, atol=1e-12), k
        else:
            assert np.array_equal(z[k], v), k


class _StubDecoder:
    """generate() by the pipeline's own model on the CPU: the text assembly around it is what is tested"""

    def __init__(self, model):
        self.model, self.calls = model, []

    def generate(self, ids, max_new_tokens, do_sample, temperature, top_k, top_p, repetition_penalty, eos_token_ids,
                 seed):
        self.calls.append(dict(max_new_tokens=max_new_tokens, do_sample=do_sample, repetition_penalty=repetition_penalty,
                               eos_token_ids=eos_token_ids, seed=seed))
        with torch.no_grad():
            out = self.model.generate(torch.tensor([ids]), max_new_tokens=max_new_tokens, do_sample=False,
                                      repetition_penalty=repetition_penalty, eos_token_id=eos_token_ids or None,
                                      pad_token_id=0)
        return out[0, len(ids):].tolist()


@pytest.mark.parametrize("from_snapshot", [True, False])
def test_pipeline_text_assembly(tmp_path, monkeypatch, from_snapshot):
    """HuggingFacePipeline around a real transformers text-generation pipeline (built as RAGHelper_local.py builds it)
    returns the pipeline's own text, for a model loaded from a snapshot and for one built in memory from its config"""
    from transformers import AutoModelForCausalLM, AutoTokenizer, LlamaForCausalLM, pipeline
    from ragmeup_b200 import llms
    model, tok = mg.save_chat_snapshot(str(tmp_path))
    if from_snapshot:
        model, tok = AutoModelForCausalLM.from_pretrained(str(tmp_path)), AutoTokenizer.from_pretrained(str(tmp_path))
    else:
        model = LlamaForCausalLM(model.config).eval()
    pipe = pipeline(model=model, tokenizer=tok, task="text-generation", temperature=0.6, repetition_penalty=1.1,
                    return_full_text=True, max_new_tokens=10)
    stub = _StubDecoder(model)
    monkeypatch.setattr(llms._PipelineGenerator, "_decoder", lambda self: stub)
    llm = llms.HuggingFacePipeline(pipeline=pipe)
    prompt = "w5 w6 w7 w8 w9 " + mg.ASSISTANT
    with torch.no_grad():
        want = pipe(prompt, do_sample=False)[0]["generated_text"]
    got = llm.invoke(prompt)
    assert got == want and got.startswith(prompt)
    assert stub.calls[0]["max_new_tokens"] == 10 and stub.calls[0]["repetition_penalty"] == pytest.approx(1.1)
    assert stub.calls[0]["eos_token_ids"] == [1]
    reply = got[got.rindex(mg.ASSISTANT) + len(mg.ASSISTANT):]
    assert reply == want[len(prompt):]
    assert llm.batch([prompt, prompt]) == [want, want]
    torch.manual_seed(7)
    llm.invoke(prompt)
    torch.manual_seed(7)
    llm.invoke(prompt)
    assert stub.calls[-1]["seed"] == stub.calls[-2]["seed"]
    with pytest.raises(ValueError, match="stop"):
        llm.invoke(prompt, stop=["w9"])
    pipe2 = pipeline(model=model, tokenizer=tok, task="text-generation", max_new_tokens=4, num_beams=2)
    with pytest.raises(ValueError, match="num_beams"):
        llms.HuggingFacePipeline(pipeline=pipe2).invoke(prompt)
