"""LLM provenance's host side: the scoring prompt per document (str and Document contexts, braces), the reply's parse
and its errors, the settings and seeds handed to the decoder, the force_cpu refusal, the oracle's agreement with the
drop-in's prompt and parse, and rmu_decoder_generate_batch's refusals that come before any CUDA call."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from oracle import llm_provenance_ref as ref
from ragmeup_b200 import provenance

PROMPT = "Q: {query} | D: {context} | A: {answer} | score 0-10"


class Doc:
    def __init__(self, text):
        self.page_content = text

    def __str__(self):
        return f"page_content='{self.page_content}'"


class Tok:
    """a stand-in tokenizer: one id per character, a chat template with a Llama-3-style tail"""
    eos_token = "<eot>"
    eos_token_id = 1

    def convert_tokens_to_ids(self, t):
        return 1 if t == "<eot>" else 0

    def apply_chat_template(self, msgs, tokenize=False):
        assert tokenize is False and len(msgs) == 1 and msgs[0]["role"] == "user"
        return "user\n\n" + msgs[0]["content"] + "assistant\n\n"

    def __call__(self, text, truncation=False):
        assert truncation
        return {"input_ids": [2] + [ord(c) for c in text]}            # a BOS, then the characters

    def decode(self, ids, skip_special_tokens=False):
        return "".join(chr(i) for i in ids if i > 2 or not skip_special_tokens)


@pytest.fixture(autouse=True)
def _env(monkeypatch):
    monkeypatch.setenv("provenance_llm_prompt", PROMPT)
    monkeypatch.delenv("force_cpu", raising=False)


def _text(ids):
    return "".join(chr(i) for i in ids[1:])


def test_prompt_for_str_and_document_contexts():
    tok = Tok()
    ids = provenance._llm_prompt(tok, "q{1}", "plain {x} text", "ans")
    assert ids[0] == 2
    assert _text(ids) == "user\n\nQ: q{1} | D: plain {x} text | A: ans | score 0-10assistant\n\n"
    d = Doc("with {braces}")
    ids = provenance._llm_prompt(tok, "q", d, "a")
    assert d.page_content == "with {{braces}}"                     # doubled in place, as the reference does
    assert "D: page_content='with {{braces}}' |" in _text(ids)
    d2 = Doc("with {braces}")
    assert ref.prompt_ids(tok, "q", d2, "a") == ids and ref.prompt_ids(tok, "q", "s", "a") == \
        provenance._llm_prompt(tok, "q", "s", "a")


def test_parse_and_its_errors():
    tok = Tok()
    ids = [2] + [ord(c) for c in "user\n\nscore 5assistant\n\n"]
    new = [ord(c) for c in "I give 7,5 then 8."]
    assert provenance._llm_score(tok, ids, new) == "8." == ref.parse(tok, ids, new)
    assert provenance._llm_score(tok, ids, [ord(c) for c in "about 7,25"]) == "7.25"
    with pytest.raises(IndexError):
        provenance._llm_score(tok, ids, [ord(c) for c in "no number"])
    with pytest.raises(ValueError):
        provenance._llm_score(tok, [2, 65], [ord("4")])


class FakeDecoder:
    def __init__(self, replies):
        self.replies = replies
        self.calls = []

    def generate_batch(self, prompts, max_new_tokens, seeds, **settings):
        self.calls.append((prompts, max_new_tokens, seeds, settings))
        return [[ord(c) for c in r] for r in self.replies]


def test_drop_in_passes_settings_and_seeds(monkeypatch):
    import torch
    from transformers import GenerationConfig
    fake = FakeDecoder(["3", "score: 9", "10"])
    monkeypatch.setattr(provenance, "_decoder", lambda model: fake)

    class Model:
        generation_config = GenerationConfig(do_sample=True, temperature=0.6, top_p=0.9, eos_token_id=[1, 9])

    tok = Tok()
    torch.manual_seed(5)
    got = provenance.compute_llm_provenance(tok, Model(), "q", ["a", Doc("b"), "c"], "ans")
    assert got == ["3", "9", "10"]
    (prompts, max_new, seeds, settings), = fake.calls                  # one call for every document
    assert max_new == 10 and len(prompts) == 3 and len(set(seeds)) == 3
    assert settings == dict(do_sample=True, temperature=0.6, top_k=50, top_p=0.9, repetition_penalty=1.0,
                            eos_token_ids=[1, 9])
    torch.manual_seed(5)
    assert [int(torch.randint(0, 2 ** 63 - 1, (1,)).item()) for _ in range(3)] == seeds
    assert tok.pad_token == "<eot>" and tok.pad_token_id == 1 and tok.eos_token_id == 1
    assert provenance.compute_llm_provenance(tok, Model(), "q", [], "ans") == []

    class Beams:
        generation_config = GenerationConfig(num_beams=4)

    with pytest.raises(ValueError, match="num_beams"):
        provenance.compute_llm_provenance(tok, Beams(), "q", ["a"], "ans")


def test_force_cpu_is_refused(monkeypatch):
    from ragmeup_b200 import _lib
    monkeypatch.setenv("force_cpu", "True")
    with pytest.raises(_lib.RmuError):
        provenance.compute_llm_provenance(Tok(), "synthetic:tiny-llama", "q", ["a"], "ans")


def test_generate_batch_refusals_before_cuda():
    from ragmeup_b200 import _lib
    L = _lib.lib()
    ids = np.zeros(4, dtype=np.int32)
    cu = np.array([0, 2, 4], dtype=np.int32)
    out = np.zeros(8, dtype=np.int32)
    n = np.zeros(2, dtype=np.int32)
    s = _lib.SamplingC(0, 1.0, 1.0, 1.0, 50, 0, (C.c_int32 * _lib.MAX_EOS)())
    assert L.rmu_decoder_generate_batch(None, ids.ctypes.data, cu.ctypes.data, 2, C.byref(s), ids.ctypes.data, 4,
                                        out.ctypes.data, n.ctypes.data, None, None) == -1
    assert b"bad argument" in L.rmu_last_error()
    assert _lib.MAX_GENERATE_BATCH == 16


def test_oracle_against_transformers_generate(tmp_path, monkeypatch):
    """the oracle's prompts and float64 greedy generation against transformers' generate on the tiny BPE chat snapshot
    (CPU, greedy), token for token, and the parse of transformers' own output"""
    import torch
    from bpe_chat_snapshot import PROMPT, save_bpe_chat_snapshot
    from oracle import generation_ref as gref
    from ragmeup_b200 import llms
    from ragmeup_b200.weights import decoder_lm_head, resolve_decoder
    model, _ = save_bpe_chat_snapshot(str(tmp_path))
    from transformers import AutoTokenizer
    tok = AutoTokenizer.from_pretrained(str(tmp_path))
    monkeypatch.setenv("provenance_llm_prompt", PROMPT)
    cfg, w = resolve_decoder(str(tmp_path))
    lm = decoder_lm_head(str(tmp_path), cfg)
    for doc in ("the first document {x}", Doc("a {second} document"), "3 5"):
        ids = ref.prompt_ids(tok, "which query", doc, "the answer 6")
        settings = llms.resolve_settings(model.generation_config, {"max_new_tokens": 10}, len(ids))
        mine = gref.generate(w, lm, cfg, ids, 10, False, penalty=settings["repetition_penalty"],
                             eos=settings["eos_token_ids"])
        with torch.no_grad():
            out = model.generate(input_ids=torch.tensor([ids]), attention_mask=torch.ones(1, len(ids), dtype=torch.long),
                                 max_new_tokens=10, do_sample=False)
        theirs = out[0, len(ids):].tolist()
        assert mine == theirs
        text = tok.decode(out[0], skip_special_tokens=True)
        assert text.count("assistant\n\n") == 1                       # the template's header, not the prompt's
        try:
            want = ref.parse(tok, ids, theirs)
        except IndexError:
            want = "IndexError"
        try:
            got = provenance._llm_score(tok, ids, mine)
        except IndexError:
            got = "IndexError"
        assert got == want
