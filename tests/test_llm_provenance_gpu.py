"""compute_llm_provenance and DecoderAttention.generate_batch on the GPU decoder against the float64 oracle
(oracle/llm_provenance_ref.py, generation_ref) on the tiny byte-level BPE chat snapshot (bpe_chat_snapshot.py), on
split and NF4 handles: the generated token ids and the parsed scores, the repeat under torch.manual_seed, the one
shared handle, and a batch above the per-call cap against per-prompt generate."""
from __future__ import annotations

import gc

import numpy as np
import pytest
import torch

from bpe_chat_snapshot import PROMPT, save_bpe_chat_snapshot
from oracle import generation_ref as gref
from oracle import llm_provenance_ref as ref
from oracle import nf4_ref as nf4

pytestmark = pytest.mark.gpu

PROJ = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj", "mlp.up_proj",
        "mlp.down_proj")


@pytest.fixture(autouse=True)
def _release_torch_cache():
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    yield


class Doc:
    def __init__(self, text):
        self.page_content = text

    def __str__(self):                                  # as langchain's Document prints: no object address
        return f"page_content='{self.page_content}'"


def _outcome(f):
    try:
        return f()
    except (IndexError, ValueError) as e:
        return type(e).__name__


CONTEXT = ["the first document {x}", "a second, longer document about the answer and the query", "third", "4 5 6"]


def _docs():
    return [CONTEXT[0], Doc(CONTEXT[1]), CONTEXT[2], Doc(CONTEXT[3])]


@pytest.mark.parametrize("weights", ["split", "nf4"])
def test_drop_in_matches_the_oracle_and_shares_the_handle(tmp_path, monkeypatch, weights):
    from transformers import AutoModelForCausalLM, AutoTokenizer
    from ragmeup_b200 import llms, provenance
    from ragmeup_b200.weights import decoder_lm_head, resolve_decoder
    save_bpe_chat_snapshot(str(tmp_path))
    model = AutoModelForCausalLM.from_pretrained(str(tmp_path)).eval()
    tok = AutoTokenizer.from_pretrained(str(tmp_path))
    monkeypatch.setenv("provenance_llm_prompt", PROMPT)
    monkeypatch.setenv("RMU_DECODER_WEIGHTS", weights)
    got = _outcome(lambda: provenance.compute_llm_provenance(tok, model, "which query", _docs(), "the answer 6"))
    dec = provenance._decoder(model)
    n = len(provenance._DECODERS)
    assert dec.weights == weights
    cfg, w = resolve_decoder(str(tmp_path))
    if weights == "nf4":                                # the weights the NF4 handle computes with
        w = {k: (nf4.nf4_weight(v) if any(k.endswith(p + ".weight") for p in PROJ) else v) for k, v in w.items()}
    lm = decoder_lm_head(str(tmp_path), cfg)
    # the generated ids, prompt by prompt, and the parsed scores
    prompts = [ref.prompt_ids(tok, "which query", d, "the answer 6") for d in _docs()]
    assert prompts == [provenance._llm_prompt(tok, "which query", d, "the answer 6") for d in _docs()]
    settings = llms.resolve_settings(model.generation_config, {"max_new_tokens": 10}, max(map(len, prompts)))
    assert not settings["do_sample"]                    # greedy: the oracle's seeds do not matter
    kw = {k: v for k, v in settings.items() if k != "max_new_tokens"}
    new = dec.generate_batch(prompts, 10, [0] * len(prompts), **kw)
    for p, ids in zip(prompts, new):
        assert ids == gref.generate(w, lm, cfg, p, 10, False, penalty=settings["repetition_penalty"],
                                    eos=settings["eos_token_ids"])
    want = _outcome(lambda: ref.compute(tok, w, lm, cfg, False, "which query", _docs(), "the answer 6", settings,
                                        [0] * len(CONTEXT)))
    assert got == want
    torch.manual_seed(3)
    a = _outcome(lambda: provenance.compute_llm_provenance(tok, model, "q", _docs(), "ans"))
    torch.manual_seed(3)
    b = _outcome(lambda: provenance.compute_llm_provenance(tok, model, "q", _docs(), "ans"))
    assert a == b
    assert provenance._decoder(model) is dec and len(provenance._DECODERS) == n   # the handle compute_attention uses


def test_generate_batch_above_the_cap_equals_per_prompt_generate(tmp_path, monkeypatch):
    """20 prompts (two calls of the C entry: 16 + 4), sampled with a penalty and eos: each equals generate"""
    from ragmeup_b200 import _lib, provenance
    save_bpe_chat_snapshot(str(tmp_path))
    dec = provenance.DecoderAttention(str(tmp_path))
    rng = np.random.default_rng(1)
    prefix = rng.integers(4, 384, 40).tolist()
    prompts = [prefix + rng.integers(4, 384, 1 + (7 * i) % 23).tolist() for i in range(20)]
    seeds = [11 * i + 3 for i in range(20)]
    kw = dict(do_sample=True, temperature=0.8, top_k=50, top_p=0.9, repetition_penalty=1.2, eos_token_ids=[1, 7])
    assert len(prompts) > _lib.MAX_GENERATE_BATCH
    got = dec.generate_batch(prompts, 8, seeds, **kw)
    assert got == [dec.generate(p, 8, seed=s, **kw) for p, s in zip(prompts, seeds)]
    with pytest.raises(ValueError):
        dec.generate_batch(prompts, 8, seeds[:3], **kw)
