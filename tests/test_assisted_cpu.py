"""Speculative decoding with a draft model without a GPU: the assistant settings HuggingFacePipeline resolves (their
transformers defaults, the assistant's own generation_config, the refusals naming their field), the
RMU_ASSISTANT_MODEL key and its conflict with prompt lookup, the settings a decoder receives from the pipeline,
compute_llm_provenance dropping them, the draft presets, and the C refusals of rmu_decoder_generate_assisted before
any CUDA call."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest


class _Assistant:
    """a transformers model as resolve_settings sees one: name_or_path and, optionally, a generation_config"""

    def __init__(self, name="synthetic:tiny-llama-draft:1", generation_config=None):
        self.name_or_path = name
        if generation_config is not None:
            self.generation_config = generation_config


def _base():
    from transformers import GenerationConfig
    from ragmeup_b200.llms import resolve_settings
    return resolve_settings(GenerationConfig(), {"max_new_tokens": 5}, 4)


def test_settings_pass_the_assistant_through_with_transformers_defaults():
    from transformers import GenerationConfig
    from ragmeup_b200.llms import resolve_settings
    base = _base()
    assert not any(k.startswith(("assistant", "num_assistant")) for k in base)
    a = _Assistant()
    got = resolve_settings(GenerationConfig(), {"max_new_tokens": 5, "assistant_model": a}, 4)
    assert got == dict(base, assistant_model=a, num_assistant_tokens=20, num_assistant_tokens_schedule="constant")
    # the assistant's own generation_config, as transformers reads it
    a = _Assistant(generation_config=GenerationConfig(num_assistant_tokens=7, num_assistant_tokens_schedule="heuristic"))
    got = resolve_settings(GenerationConfig(), {"max_new_tokens": 5, "assistant_model": a}, 4)
    assert got["num_assistant_tokens"] == 7 and got["num_assistant_tokens_schedule"] == "heuristic"
    a = _Assistant(generation_config=GenerationConfig(num_assistant_tokens_schedule="heuristic_transient",
                                                      assistant_confidence_threshold=0.9))
    got = resolve_settings(GenerationConfig(), {"max_new_tokens": 5, "assistant_model": a}, 4)
    assert got["num_assistant_tokens"] == 20 and got["num_assistant_tokens_schedule"] == "heuristic_transient"
    # the confidence threshold only ends drafting early: accepted on the target's config too, and not passed on
    got = resolve_settings(GenerationConfig(assistant_confidence_threshold=0.1), {"max_new_tokens": 5}, 4)
    assert got == base


def test_settings_refusals_name_their_field():
    from transformers import GenerationConfig
    from ragmeup_b200.llms import resolve_settings
    for bad in (object(), "synthetic:tiny-llama-draft", 3, _Assistant(name="")):
        with pytest.raises(ValueError, match="assistant_model"):
            resolve_settings(GenerationConfig(), {"assistant_model": bad}, 4)
    with pytest.raises(ValueError, match="assistant_tokenizer"):
        resolve_settings(GenerationConfig(), {"assistant_model": _Assistant(), "assistant_tokenizer": object()}, 4)

    class Cfg:
        num_assistant_tokens, num_assistant_tokens_schedule = 5, "fast"
    with pytest.raises(ValueError, match="num_assistant_tokens_schedule"):
        resolve_settings(GenerationConfig(), {"assistant_model": _Assistant(generation_config=Cfg())}, 4)
    Cfg.num_assistant_tokens_schedule, Cfg.num_assistant_tokens = "constant", -2
    with pytest.raises(ValueError, match="num_assistant_tokens"):
        resolve_settings(GenerationConfig(), {"assistant_model": _Assistant(generation_config=Cfg())}, 4)


def test_assistant_env_and_the_lookup_conflict(monkeypatch):
    from transformers import GenerationConfig
    from ragmeup_b200 import llms
    monkeypatch.delenv(llms.PROMPT_LOOKUP_ENV, raising=False)
    for raw, want in (("", None), ("  ", None), ("synthetic:tiny-llama-draft:1", "synthetic:tiny-llama-draft:1"),
                      (" /models/Llama-3.2-3B-Instruct ", "/models/Llama-3.2-3B-Instruct")):
        monkeypatch.setenv(llms.ASSISTANT_ENV, raw)
        assert llms.assistant_model_name() == want
    monkeypatch.delenv(llms.ASSISTANT_ENV)
    assert llms.assistant_model_name() is None
    base = llms.pipeline_settings(GenerationConfig(), {"max_new_tokens": 5}, 4)
    assert base == _base()
    monkeypatch.setenv(llms.ASSISTANT_ENV, "synthetic:tiny-llama-draft:1")
    got = llms.pipeline_settings(GenerationConfig(), {"max_new_tokens": 5}, 4)
    assert got["assistant_model"].name_or_path == "synthetic:tiny-llama-draft:1"
    assert got["num_assistant_tokens"] == 20 and got["num_assistant_tokens_schedule"] == "constant"
    # the kwargs' assistant wins over the key
    a = _Assistant(name="synthetic:tiny-llama:3")
    assert llms.pipeline_settings(GenerationConfig(), {"max_new_tokens": 5, "assistant_model": a}, 4)[
        "assistant_model"] is a
    # prompt lookup and a draft model both on, from any source
    for lookup_env, kwargs in (("4", {}), ("", {"prompt_lookup_num_tokens": 3})):
        monkeypatch.setenv(llms.PROMPT_LOOKUP_ENV, lookup_env)
        with pytest.raises(ValueError, match="prompt_lookup_num_tokens.*assistant_model"):
            llms.pipeline_settings(GenerationConfig(), dict(kwargs, max_new_tokens=5), 4)
    monkeypatch.delenv(llms.ASSISTANT_ENV)
    monkeypatch.setenv(llms.PROMPT_LOOKUP_ENV, "2")
    with pytest.raises(ValueError, match="prompt_lookup_num_tokens.*assistant_model"):
        llms.pipeline_settings(GenerationConfig(), {"max_new_tokens": 5, "assistant_model": a}, 4)


class _StubDecoder:
    def __init__(self):
        self.calls = []

    def generate(self, ids, **kw):
        self.calls.append(kw)
        return [1]

    def generate_batch(self, prompts, max_new, seeds, **kw):
        self.calls.append(kw)
        return [[] for _ in prompts]


def test_pipeline_passes_the_draft_handle_and_provenance_drops_it(tmp_path, monkeypatch):
    """HuggingFacePipeline resolves assistant_model (or RMU_ASSISTANT_MODEL) to its own decoder handle and passes it
    with the settings; the target's own handle is refused; compute_llm_provenance's batched path drops them"""
    import make_golden_generate as mg
    from transformers import AutoModelForCausalLM, pipeline
    from ragmeup_b200 import llms, provenance
    model, tok = mg.save_chat_snapshot(str(tmp_path / "target"))
    mg.save_chat_snapshot(str(tmp_path / "draft"))
    draft_model = AutoModelForCausalLM.from_pretrained(str(tmp_path / "draft"))
    draft_model.generation_config.num_assistant_tokens = 9
    target, draft = _StubDecoder(), _StubDecoder()
    handles = {str(tmp_path / "draft"): draft, "synthetic:tiny-llama-draft:1": draft}

    def resolve(m):
        name = m if isinstance(m, str) else m.name_or_path
        return handles.get(name, target)
    monkeypatch.setattr(provenance, "_decoder", resolve)
    monkeypatch.delenv(llms.PROMPT_LOOKUP_ENV, raising=False)
    monkeypatch.delenv(llms.ASSISTANT_ENV, raising=False)
    prompt = "w5 w6 w7 " + mg.ASSISTANT
    pipe = pipeline(model=model, tokenizer=tok, task="text-generation", max_new_tokens=4, assistant_model=draft_model)
    llms.HuggingFacePipeline(pipeline=pipe).invoke(prompt)
    kw = target.calls[-1]
    assert kw["assistant"] is draft and kw["num_assistant_tokens"] == 9
    assert kw["num_assistant_tokens_schedule"] == "constant" and "assistant_model" not in kw
    plain = pipeline(model=model, tokenizer=tok, task="text-generation", max_new_tokens=4)
    llms.HuggingFacePipeline(pipeline=plain).invoke(prompt)
    assert "assistant" not in target.calls[-1]
    monkeypatch.setenv(llms.ASSISTANT_ENV, "synthetic:tiny-llama-draft:1")
    llms.HuggingFacePipeline(pipeline=plain).invoke(prompt)
    assert target.calls[-1]["assistant"] is draft and target.calls[-1]["num_assistant_tokens"] == 20
    monkeypatch.setenv(llms.ASSISTANT_ENV, str(tmp_path / "target"))         # the target's own handle
    with pytest.raises(ValueError, match="assistant_model.*target's own decoder"):
        llms.HuggingFacePipeline(pipeline=plain).invoke(prompt)
    monkeypatch.delenv(llms.ASSISTANT_ENV)
    model.generation_config.prompt_lookup_num_tokens = None
    monkeypatch.setattr(provenance, "_llm_prompt", lambda tokenizer, q, d, a: [1, 2, 3])
    monkeypatch.setattr(provenance, "_llm_score", lambda tokenizer, p, n: "1")
    import ragmeup_b200.llms as L

    real = L.resolve_settings
    monkeypatch.setattr(L, "resolve_settings",
                        lambda gc, kw, n: real(gc, dict(kw, assistant_model=draft_model), n))
    provenance.compute_llm_provenance(tok, model, "q", ["doc"], "answer")
    assert not any(k.startswith(("assistant", "num_assistant")) for k in target.calls[-1])


def test_decoder_attention_refuses_two_drafters():
    from ragmeup_b200 import provenance
    dec = provenance.DecoderAttention.__new__(provenance.DecoderAttention)
    dec.cfg = type("Cfg", (), {"name": "synthetic:tiny-llama"})()
    with pytest.raises(ValueError, match="prompt_lookup_num_tokens and assistant"):
        dec.generate([1, 2], 4, assistant=object(), prompt_lookup_num_tokens=3)


def test_draft_presets():
    from ragmeup_b200.weights import DECODER_PRESETS, LlamaConfig, Qwen3Config, decoder_config
    p = DECODER_PRESETS["llama-3.2-3b"]
    assert isinstance(p, LlamaConfig)
    assert (p.hidden, p.layers, p.heads, p.kv_heads, p.ffn, p.vocab_size) == (3072, 28, 24, 8, 8192, 128256)
    assert p.hidden // p.heads == 128 and p.rope_scaling[0] == 32.0
    q = DECODER_PRESETS["qwen3-0.6b"]
    assert isinstance(q, Qwen3Config) and q.tie_word_embeddings
    assert (q.hidden, q.layers, q.heads, q.kv_heads, q.head_dim, q.ffn, q.vocab_size) == (1024, 28, 16, 8, 128, 3072,
                                                                                           151936)
    assert q.vocab_size == DECODER_PRESETS["qwen3-32b"].vocab_size
    assert p.vocab_size == DECODER_PRESETS["llama-3.1-8b"].vocab_size == DECODER_PRESETS["llama-3.1-70b"].vocab_size
    t = decoder_config("synthetic:tiny-llama-draft:3")
    tiny = DECODER_PRESETS["tiny-llama"]
    assert (t.layers, t.heads, t.kv_heads, t.vocab_size) == (1, 2, 1, tiny.vocab_size)
    assert (t.rope_theta, t.rope_scaling) == (tiny.rope_theta, tiny.rope_scaling)


def test_c_refusals_before_any_cuda_call():
    from ragmeup_b200 import _lib
    L = _lib.lib()
    s = _lib.SamplingC(0, 1.0, 1.0, 1.0, 0, 0, (C.c_int32 * _lib.MAX_EOS)())
    out = np.zeros(4, np.int32)
    n = C.c_int32()
    ids = np.zeros(3, np.int32)
    fake_a, fake_b = np.zeros(64, np.uint8), np.zeros(64, np.uint8)   # never dereferenced by these refusals
    a, b = fake_a.ctypes.data, fake_b.ctypes.data

    def call(enc, draft, num_tokens=3, schedule=0, T=3):
        return L.rmu_decoder_generate_assisted(enc, draft, ids.ctypes.data, T, C.byref(s), 0, 4, num_tokens, schedule,
                                               out.ctypes.data, C.byref(n), None, None, None, None, None)
    assert call(None, b) == -1
    assert call(a, None) == -1
    assert call(a, b, num_tokens=-1) == -1
    assert call(a, b, T=0) == -1
    assert call(a, b, schedule=2) == -1 and b"schedule" in L.rmu_last_error()
    assert call(a, b, schedule=-1) == -1
    assert call(a, a) == -1 and b"another handle" in L.rmu_last_error()
