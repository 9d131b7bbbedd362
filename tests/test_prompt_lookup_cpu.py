"""Prompt-lookup decoding without a GPU: the host drafter (rmu_prompt_lookup_draft) against transformers'
PromptLookupCandidateGenerator, the fact that makes the setting a pure speed choice (transformers' greedy generate with
prompt_lookup_num_tokens gives plain generate's ids, in float64), the settings HuggingFacePipeline resolves and the
environment key, and the C refusals of the new entry points."""
from __future__ import annotations

import ctypes as C
from dataclasses import replace

import numpy as np
import pytest
import torch

from ragmeup_b200.weights import DECODER_PRESETS, synthetic_llama_weights


def _draft(ids, k, ngram, max_len):
    from ragmeup_b200 import _lib
    a = np.ascontiguousarray(ids, dtype=np.int32)
    out = np.full(max(k, 1), -9, dtype=np.int32)
    n = _lib.lib().rmu_prompt_lookup_draft(a.ctypes.data, len(a), k, ngram, max_len, out.ctypes.data)
    assert n >= 0
    assert (out[n:] == -9).all()
    return out[:n].tolist()


def _want(ids, k, ngram, max_len):
    from transformers.generation.candidate_generator import PromptLookupCandidateGenerator
    g = PromptLookupCandidateGenerator(eos_token_id=torch.tensor([-1]), num_output_tokens=k,
                                       max_matching_ngram_size=ngram, max_length=max_len)
    x = torch.tensor([ids], dtype=torch.long)
    cand, _ = g.get_candidates(x)
    return cand[0, len(ids):].tolist()


def _sequences():
    rng = np.random.default_rng(0)
    out = [rng.integers(0, 50, n).tolist() for n in (1, 2, 3, 8, 40, 200)]             # random
    out += [rng.integers(0, 6, 60).tolist()]                                            # many short matches
    out += [([1, 2, 3, 4, 5] * 12)[:m] for m in (5, 6, 11, 33, 60)]                     # periodic
    out += [[7] * 30, [7] * 29 + [8], [1, 2] * 10 + [3, 1, 2], [9, 9, 1, 9, 9]]        # runs, a last n-gram seen once
    out += [[4, 5, 6, 0, 4, 5], [4, 5, 0, 4, 5]]                                        # matches at the very end
    return out


@pytest.mark.parametrize("ngram", [1, 2, 3, 4])
def test_drafter_matches_transformers(ngram):
    for ids in _sequences():
        for k in (1, 2, 3, 7, 15):
            for max_len in (len(ids) + 1, len(ids) + 2, len(ids) + 5, len(ids) + 100, len(ids) - 1):
                assert _draft(ids, k, ngram, max_len) == _want(ids, k, ngram, max_len), (ids, k, ngram, max_len)


def test_drafter_refusals():
    from ragmeup_b200 import _lib
    L = _lib.lib()
    a = np.zeros(4, np.int32)
    assert L.rmu_prompt_lookup_draft(None, 4, 2, 2, 10, a.ctypes.data) == -1
    assert L.rmu_prompt_lookup_draft(a.ctypes.data, 4, 2, 2, 10, None) == -1
    assert L.rmu_prompt_lookup_draft(a.ctypes.data, 0, 2, 2, 10, a.ctypes.data) == -1
    assert L.rmu_prompt_lookup_draft(a.ctypes.data, 4, 0, 2, 10, a.ctypes.data) == -1
    assert L.rmu_prompt_lookup_draft(a.ctypes.data, 4, 2, 0, 10, a.ctypes.data) == -1


def test_transformers_prompt_lookup_keeps_greedy_ids():
    """transformers' own prompt-lookup decoding in float64 returns plain greedy generate's ids, with a prompt whose
    repeats make the lookups hit"""
    from transformers import LlamaConfig as HC, LlamaForCausalLM
    cfg = replace(DECODER_PRESETS["tiny-llama"], layers=2, max_pos=128)
    w = synthetic_llama_weights(cfg, seed=1, scale=4.0)
    rs = cfg.rope_scaling
    hc = HC(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, intermediate_size=cfg.ffn, num_hidden_layers=cfg.layers,
            num_attention_heads=cfg.heads, num_key_value_heads=cfg.kv_heads, head_dim=128,
            max_position_embeddings=cfg.max_pos, rms_norm_eps=cfg.ln_eps, rope_theta=cfg.rope_theta,
            rope_scaling={"rope_type": "llama3", "factor": rs[0], "low_freq_factor": rs[1], "high_freq_factor": rs[2],
                          "original_max_position_embeddings": rs[3], "rope_theta": cfg.rope_theta},
            tie_word_embeddings=False)
    lm = (np.random.default_rng(2).standard_normal((cfg.vocab_size, cfg.hidden)) * 0.5).astype(np.float32)
    model = LlamaForCausalLM(hc).to(torch.float64).eval()
    sd = {"model." + k: torch.tensor(v, dtype=torch.float64) for k, v in w.items()}
    sd["lm_head.weight"] = torch.tensor(lm, dtype=torch.float64)
    model.load_state_dict(sd, strict=False)
    span = [5, 17, 3, 250, 9, 41, 77, 12]
    ids = torch.tensor([span + [600, 601] + span + [602] + span[:3]])
    with torch.no_grad():
        plain = model.generate(ids, max_new_tokens=12, do_sample=False, pad_token_id=0, eos_token_id=999)
        for k in (1, 3, 10):
            got = model.generate(ids, max_new_tokens=12, do_sample=False, pad_token_id=0, eos_token_id=999,
                                 prompt_lookup_num_tokens=k)
            assert got.tolist() == plain.tolist(), k


def test_settings_pass_lookup_through_only_when_on():
    from transformers import GenerationConfig
    from ragmeup_b200.llms import resolve_settings
    base = resolve_settings(GenerationConfig(), {"max_new_tokens": 5}, 4)
    assert "prompt_lookup_num_tokens" not in base and "max_matching_ngram_size" not in base
    assert resolve_settings(GenerationConfig(), {"max_new_tokens": 5, "prompt_lookup_num_tokens": 0}, 4) == base
    on = resolve_settings(GenerationConfig(), {"max_new_tokens": 5, "prompt_lookup_num_tokens": 7}, 4)
    assert on == dict(base, prompt_lookup_num_tokens=7, max_matching_ngram_size=2)
    on = resolve_settings(GenerationConfig(prompt_lookup_num_tokens=3, max_matching_ngram_size=4), {"max_new_tokens": 5}, 4)
    assert on == dict(base, prompt_lookup_num_tokens=3, max_matching_ngram_size=4)
    with pytest.raises(ValueError, match="assistant_model"):
        resolve_settings(GenerationConfig(), {"assistant_model": object()}, 4)


def test_prompt_lookup_env(monkeypatch):
    from ragmeup_b200 import llms
    monkeypatch.delenv(llms.PROMPT_LOOKUP_ENV, raising=False)
    assert llms.prompt_lookup_tokens() == 0
    for raw, want in (("0", 0), ("10", 10), (" 3 ", 3), ("", 0)):
        monkeypatch.setenv(llms.PROMPT_LOOKUP_ENV, raw)
        assert llms.prompt_lookup_tokens() == want
    for raw in ("-1", "two", "1.5"):
        monkeypatch.setenv(llms.PROMPT_LOOKUP_ENV, raw)
        with pytest.raises(ValueError, match=llms.PROMPT_LOOKUP_ENV):
            llms.prompt_lookup_tokens()


class _StubDecoder:
    def __init__(self):
        self.calls = []

    def generate(self, ids, **kw):
        self.calls.append(kw)
        return [1]

    def generate_batch(self, prompts, max_new, seeds, **kw):
        self.calls.append(kw)
        return [[] for _ in prompts]


def test_pipeline_default_from_env_and_provenance_drops_keys(tmp_path, monkeypatch):
    """the env key fills in prompt_lookup_num_tokens only when the pipeline does not set it; compute_llm_provenance's
    batched path never passes the keys on"""
    import make_golden_generate as mg
    from transformers import pipeline
    from ragmeup_b200 import llms, provenance
    model, tok = mg.save_chat_snapshot(str(tmp_path))
    stub = _StubDecoder()
    monkeypatch.setattr(llms._PipelineGenerator, "_decoder", lambda self: stub)
    prompt = "w5 w6 w7 " + mg.ASSISTANT
    pipe = pipeline(model=model, tokenizer=tok, task="text-generation", max_new_tokens=4)
    monkeypatch.delenv(llms.PROMPT_LOOKUP_ENV, raising=False)
    llms.HuggingFacePipeline(pipeline=pipe).invoke(prompt)
    assert "prompt_lookup_num_tokens" not in stub.calls[-1]
    monkeypatch.setenv(llms.PROMPT_LOOKUP_ENV, "0")
    llms.HuggingFacePipeline(pipeline=pipe).invoke(prompt)
    assert "prompt_lookup_num_tokens" not in stub.calls[-1]
    monkeypatch.setenv(llms.PROMPT_LOOKUP_ENV, "6")
    llms.HuggingFacePipeline(pipeline=pipe).invoke(prompt)
    assert stub.calls[-1]["prompt_lookup_num_tokens"] == 6 and stub.calls[-1]["max_matching_ngram_size"] == 2
    pipe3 = pipeline(model=model, tokenizer=tok, task="text-generation", max_new_tokens=4, prompt_lookup_num_tokens=3)
    llms.HuggingFacePipeline(pipeline=pipe3).invoke(prompt)
    assert stub.calls[-1]["prompt_lookup_num_tokens"] == 3
    monkeypatch.setenv(llms.PROMPT_LOOKUP_ENV, "x")
    with pytest.raises(ValueError, match=llms.PROMPT_LOOKUP_ENV):
        llms.HuggingFacePipeline(pipeline=pipe).invoke(prompt)
    model.generation_config.prompt_lookup_num_tokens = 5
    monkeypatch.setattr(provenance, "_decoder", lambda m: stub)
    monkeypatch.setattr(provenance, "_llm_prompt", lambda tokenizer, q, d, a: [1, 2, 3])
    monkeypatch.setattr(provenance, "_llm_score", lambda tokenizer, p, n: "1")
    provenance.compute_llm_provenance(tok, model, "q", ["doc"], "answer")
    assert "prompt_lookup_num_tokens" not in stub.calls[-1] and "max_matching_ngram_size" not in stub.calls[-1]


def test_c_refusals():
    from ragmeup_b200 import _lib
    L = _lib.lib()
    s = _lib.SamplingC(0, 1.0, 1.0, 1.0, 0, 0, (C.c_int32 * _lib.MAX_EOS)())
    out = np.zeros(4, np.int32)
    n, passes = C.c_int32(), C.c_int32()
    ids = np.zeros(3, np.int32)
    assert L.rmu_decoder_generate_lookup(None, ids.ctypes.data, 3, C.byref(s), 0, 4, 2, 2, out.ctypes.data, C.byref(n),
                                         None, C.byref(passes), None) == -1
    assert L.rmu_debug_generate_drafts(None, ids.ctypes.data, 3, C.byref(s), 0, 4, ids.ctypes.data, 2, out.ctypes.data,
                                       C.byref(n), None, C.byref(passes), None) == -1
    x = np.zeros(64, np.float32)
    assert L.rmu_debug_sample_verify_rows(x.ctypes.data, 8, 17, x.ctypes.data, x.ctypes.data, 0, 0, C.byref(s),
                                          x.ctypes.data, x.ctypes.data, None) == -1               # M above 16
    assert L.rmu_debug_sample_verify_rows(x.ctypes.data, 8, 2, x.ctypes.data, x.ctypes.data, 0, -1, C.byref(s),
                                          x.ctypes.data, x.ctypes.data, None) == -1               # step0 < 0
    s.do_sample = 1                                                                            # top_k 0 when sampling
    assert L.rmu_debug_sample_verify_rows(x.ctypes.data, 8, 2, x.ctypes.data, x.ctypes.data, 0, 0, C.byref(s),
                                          x.ctypes.data, x.ctypes.data, None) == -3

