"""``HuggingFacePipeline`` — langchain's LLM wrapper around a transformers ``text-generation`` pipeline, with the
model's ``generate`` on the GPU decoder (SURVEY.md §3.1: the chat model's replies are the reference's dominant wall
time; ``server/RAGHelper_local.py:105`` builds the wrapper).

Opt in by import, as attention provenance is: ``from ragmeup_b200.llms import HuggingFacePipeline`` in place of
``from langchain_huggingface.llms import HuggingFacePipeline``.  Only ``generate`` is replaced:

* the prompt is tokenised by the caller's pipeline (``preprocess`` with its ``_preprocess_params``), and the returned
  text is built by the caller's ``postprocess`` (its ``_postprocess_params``), so both are whatever the installed
  transformers does;
* the decoder is found from ``pipeline.model.name_or_path`` as ``provenance.compute_attention`` finds it, and shares
  ``provenance._DECODERS`` with it: one upload of the weights per (snapshot, device);
* the settings are ``pipeline.generation_config`` updated with the pipeline's generate kwargs, transformers' defaults
  for what is unset.  A setting the sampler does not compute raises a ``ValueError`` naming the field;
* the seed is drawn from torch's CPU default generator, so ``torch.manual_seed`` makes a run repeat (the draw itself is
  an inverse CDF over a Philox uniform, not ``torch.multinomial``: no parity with torch's random stream).

The model the pipeline holds (the reference's NF4 model) stays loaded but generates nothing.
"""
from __future__ import annotations

import copy
import os
import threading
from concurrent.futures import ThreadPoolExecutor
from typing import Any, List, Optional

from . import provenance

# GenerationConfig fields the GPU sampler does not compute: each must keep transformers' default value
REFUSED_FIELDS = ("num_beams", "num_beam_groups", "num_return_sequences", "min_p", "typical_p", "no_repeat_ngram_size",
                  "bad_words_ids", "sequence_bias", "suppress_tokens", "begin_suppress_tokens", "forced_bos_token_id",
                  "forced_eos_token_id", "min_new_tokens", "min_length", "stop_strings", "epsilon_cutoff", "eta_cutoff",
                  "guidance_scale", "encoder_repetition_penalty", "encoder_no_repeat_ngram_size", "diversity_penalty",
                  "exponential_decay_length_penalty", "renormalize_logits", "constraints", "force_words_ids",
                  "penalty_alpha", "watermarking_config", "top_h", "dola_layers")
# unset fields hold None in a GenerationConfig built from scratch and False / 0 / [] in one built from a model's config:
# these values all mean "off"


def _off(v) -> bool:
    return v is None or v is False or (not isinstance(v, bool) and isinstance(v, (int, float)) and v == 0) or v == [] \
        or v == {}


def resolve_settings(generation_config: Any, generate_kwargs: dict, prompt_len: int) -> dict:
    """``generation_config`` (a transformers GenerationConfig) updated with ``generate_kwargs``, transformers' defaults
    for the fields left unset -> the arguments of ``DecoderAttention.generate``; ValueError naming the first field the
    sampler does not compute"""
    from transformers import GenerationConfig
    gc = copy.deepcopy(generation_config) if generation_config is not None else GenerationConfig()
    generate_kwargs = dict(generate_kwargs)
    assistant = generate_kwargs.pop("assistant_model", None)
    if generate_kwargs.pop("assistant_tokenizer", None) is not None:
        raise ValueError("generate kwarg 'assistant_tokenizer' is not supported by the GPU decoder: the draft model must "
                         "share the target's tokenizer (universal assisted decoding is not computed)")
    unused = gc.update(**generate_kwargs)
    if unused:
        raise ValueError(f"generate kwarg {sorted(unused)[0]!r} is not supported by the GPU decoder")
    defaults = GenerationConfig._get_default_generation_params()

    def get(field):
        v = getattr(gc, field, None)
        return defaults.get(field) if v is None else v

    for field in REFUSED_FIELDS:
        v, d = get(field), defaults.get(field)
        if v != d and not (_off(v) and _off(d)):
            raise ValueError(f"generation setting {field} = {get(field)!r} is not supported by the GPU decoder's sampler")
    do_sample = bool(get("do_sample"))
    top_k = get("top_k")
    if do_sample and not (top_k and 1 <= int(top_k) <= 256):
        raise ValueError(f"generation setting top_k = {top_k!r} is not supported when sampling: the sampler keeps at "
                         f"most 256 candidates (1 <= top_k <= 256)")
    eos = gc.eos_token_id
    eos = [] if eos is None else ([int(eos)] if isinstance(eos, int) else [int(t) for t in eos])
    max_new = gc.max_new_tokens if gc.max_new_tokens is not None else int(get("max_length")) - int(prompt_len)
    out = dict(max_new_tokens=int(max_new), do_sample=do_sample, temperature=float(get("temperature")),
               top_k=int(top_k or 0), top_p=float(get("top_p")), repetition_penalty=float(get("repetition_penalty")),
               eos_token_ids=eos)
    lookup = get("prompt_lookup_num_tokens")
    if not _off(lookup):
        # prompt-lookup decoding changes how many passes a reply takes, never its tokens
        out.update(prompt_lookup_num_tokens=int(lookup), max_matching_ngram_size=int(get("max_matching_ngram_size") or 2))
    if assistant is not None:
        out.update(assistant_settings(assistant))
    return out


def assistant_settings(assistant: Any) -> dict:
    """``assistant_model`` (a transformers model with ``name_or_path``, or a ``provenance.DecoderAttention``) -> the
    draft settings ``HuggingFacePipeline`` passes on: the model itself and, as transformers reads them, the drafts per
    pass and their schedule from the assistant's own ``generation_config`` (transformers' defaults, 20 and
    ``"constant"``, without one).  Speculative decoding changes how many passes a reply takes, never its tokens.
    ``assistant_confidence_threshold`` only ends drafting early, so it is accepted and not computed.  ValueError naming
    ``assistant_model`` for anything else, and naming the setting for a count or schedule the drafter does not take."""
    if not isinstance(assistant, provenance.DecoderAttention) and not getattr(assistant, "name_or_path", None):
        raise ValueError(f"generation setting assistant_model = {assistant!r} is not supported by the GPU decoder: "
                         f"pass a transformers model with name_or_path or a DecoderAttention")
    gc = getattr(assistant, "generation_config", None)
    num = getattr(gc, "num_assistant_tokens", None)
    schedule = getattr(gc, "num_assistant_tokens_schedule", None)
    num = 20 if num is None else num
    schedule = "constant" if schedule is None else schedule
    if isinstance(num, bool) or not isinstance(num, (int, float)) or num < 0 or int(num) != num:
        raise ValueError(f"generation setting num_assistant_tokens = {num!r}: expected a non-negative integer")
    if schedule not in provenance.ASSIST_SCHEDULES:
        raise ValueError(f"generation setting num_assistant_tokens_schedule = {schedule!r} is not supported by the GPU "
                         f"decoder (one of {tuple(provenance.ASSIST_SCHEDULES)})")
    return dict(assistant_model=assistant, num_assistant_tokens=int(num), num_assistant_tokens_schedule=schedule)


PROMPT_LOOKUP_ENV = "RMU_PROMPT_LOOKUP_TOKENS"


def prompt_lookup_tokens() -> int:
    """``$RMU_PROMPT_LOOKUP_TOKENS``: the drafts per pass HuggingFacePipeline proposes when neither its generate kwargs
    nor its generation_config set ``prompt_lookup_num_tokens`` (the reference builds its pipeline with fixed kwargs, so
    its ``.env`` is where the setting can come from); unset or 0: off.  ValueError naming the key otherwise."""
    raw = os.environ.get(PROMPT_LOOKUP_ENV, "").strip()
    if not raw:
        return 0
    try:
        v = int(raw)
    except ValueError:
        v = -1
    if v < 0:
        raise ValueError(f"{PROMPT_LOOKUP_ENV}={os.environ[PROMPT_LOOKUP_ENV]!r}: expected a non-negative integer")
    return v


ASSISTANT_ENV = "RMU_ASSISTANT_MODEL"


def assistant_model_name() -> Optional[str]:
    """``$RMU_ASSISTANT_MODEL``: the draft model (a snapshot name or ``synthetic:<preset>``) HuggingFacePipeline drafts
    with when neither its generate kwargs nor its generation_config set ``assistant_model``, as
    ``RMU_PROMPT_LOOKUP_TOKENS`` does for prompt lookup; unset or empty: none"""
    return os.environ.get(ASSISTANT_ENV, "").strip() or None


class _EnvAssistant:
    """the draft model ``$RMU_ASSISTANT_MODEL`` names, as ``assistant_settings`` takes one: no generation_config, so
    transformers' defaults apply"""

    def __init__(self, name: str):
        self.name_or_path = name


def pipeline_settings(generation_config: Any, generate_kwargs: dict, prompt_len: int) -> dict:
    """``resolve_settings`` with the ``.env`` keys filled in where neither the kwargs nor the generation config set
    their field: ``RMU_PROMPT_LOOKUP_TOKENS`` and ``RMU_ASSISTANT_MODEL``.  Prompt lookup and a draft model both on,
    from any source, raise ValueError naming both."""
    settings = resolve_settings(generation_config, generate_kwargs, prompt_len)
    if "prompt_lookup_num_tokens" not in settings and prompt_lookup_tokens():
        settings.update(prompt_lookup_num_tokens=prompt_lookup_tokens(), max_matching_ngram_size=2)
    if "assistant_model" not in settings and assistant_model_name():
        settings.update(assistant_settings(_EnvAssistant(assistant_model_name())))
    if "prompt_lookup_num_tokens" in settings and "assistant_model" in settings:
        raise ValueError(f"prompt_lookup_num_tokens ({PROMPT_LOOKUP_ENV}) and assistant_model ({ASSISTANT_ENV}) are both "
                         f"set: the GPU decoder drafts from one source per reply")
    return settings


class _PipelineGenerator:
    """the parts shared by both forms of HuggingFacePipeline"""

    def _setup(self, pipeline: Any) -> None:
        self._pipe = pipeline
        self._lock = threading.Lock()

    def _decoder(self):
        return provenance._decoder(self._pipe.model)

    def _assistant(self, model: Any, target: Any):
        """the draft handle of ``model``, found as the target's is (``provenance._decoder``: the same
        ``RMU_DECODER_WEIGHTS``, memory plan and release rule); ValueError when it is the target's own handle"""
        draft = provenance._decoder(model)
        if draft is target:
            raise ValueError(f"assistant_model {getattr(model, 'name_or_path', model)!r} resolves to the target's own "
                             f"decoder: the draft must be another model")
        return draft

    def _call(self, prompt: str, seed: Optional[int] = None) -> str:
        import torch
        pipe = self._pipe
        # the lock covers the pipeline's own tokenizer and post-processing; generation runs outside it, so calls from
        # several threads share the decoder's session and their replies progress together
        with self._lock:
            inputs = pipe.preprocess(prompt, **pipe._preprocess_params)
            ids = inputs["input_ids"]
            if ids.shape[0] != 1:
                raise ValueError("one prompt per call: batched generation is not supported")
            fwd = {k: v for k, v in pipe._forward_params.items() if k not in ("generation_config",)}
            gen_cfg = pipe._forward_params.get("generation_config", getattr(pipe, "generation_config", None) or
                                               pipe.model.generation_config)
            settings = pipeline_settings(gen_cfg, fwd, ids.shape[1])
            if seed is None:
                seed = int(torch.randint(0, 2 ** 63 - 1, (1,)).item())
        dec = self._decoder()
        if "assistant_model" in settings:
            settings["assistant"] = self._assistant(settings.pop("assistant_model"), dec)
        new = dec.generate(ids[0].tolist(), seed=seed, **settings)
        with self._lock:
            seq = torch.cat([ids[0].cpu(), torch.as_tensor(new, dtype=ids.dtype)])
            model_outputs = {"generated_sequence": seq.view(1, 1, -1), "input_ids": ids,
                             "prompt_text": inputs.get("prompt_text", prompt)}
            out = pipe.postprocess(model_outputs, **pipe._postprocess_params)
        return out[0]["generated_text"] if isinstance(out[0], dict) else out[0][0]["generated_text"]

    def _call_all(self, prompts: List[str]) -> List[str]:
        """``_call`` on every prompt, all of them generating at once (one thread each), in prompt order; the seeds are
        drawn in prompt order first, so torch.manual_seed repeats a batch as it repeats a call, and the workers run on
        the caller's current CUDA device, which picks the decoder as a call on the caller's thread would"""
        import torch
        if len(prompts) <= 1:
            return [self._call(p) for p in prompts]
        seeds = [int(torch.randint(0, 2 ** 63 - 1, (1,)).item()) for _ in prompts]
        device = torch.cuda.current_device() if torch.cuda.is_available() else None

        def call(prompt, seed):
            if device is None:
                return self._call(prompt, seed)
            with torch.cuda.device(device):
                return self._call(prompt, seed)

        with ThreadPoolExecutor(max_workers=min(len(prompts), 64)) as pool:
            return list(pool.map(call, prompts, seeds))


try:
    from langchain_core.language_models.llms import BaseLLM
    from langchain_core.outputs import Generation, LLMResult

    class HuggingFacePipeline(BaseLLM, _PipelineGenerator):
        """langchain ``BaseLLM`` around a transformers text-generation pipeline; ``generate`` on the GPU decoder"""
        pipeline: Any = None

        def __init__(self, pipeline: Any = None, **kwargs):
            super().__init__(pipeline=pipeline, **kwargs)
            self._setup(pipeline)

        @property
        def _llm_type(self) -> str:
            return "ragmeup_b200_huggingface_pipeline"

        def _generate(self, prompts: List[str], stop: Optional[List[str]] = None, run_manager: Any = None,
                      **kwargs: Any) -> LLMResult:
            if stop is not None:
                raise ValueError("stop sequences are not supported by the GPU decoder")
            return LLMResult(generations=[[Generation(text=t)] for t in self._call_all(list(prompts))])

except ImportError:
    class HuggingFacePipeline(_PipelineGenerator):
        """a transformers text-generation pipeline with ``generate`` on the GPU decoder (``invoke`` / ``batch``, as
        langchain's wrapper offers them)"""

        def __init__(self, pipeline: Any = None, **kwargs):
            self.pipeline = pipeline
            self._setup(pipeline)

        def invoke(self, prompt: Any, stop: Optional[List[str]] = None, **kwargs: Any) -> str:
            if stop is not None:
                raise ValueError("stop sequences are not supported by the GPU decoder")
            return self._call(prompt.to_string() if hasattr(prompt, "to_string") else str(prompt))

        def batch(self, prompts: List[Any], **kwargs: Any) -> List[str]:
            if kwargs.get("stop") is not None:
                raise ValueError("stop sequences are not supported by the GPU decoder")
            return self._call_all([p.to_string() if hasattr(p, "to_string") else str(p) for p in prompts])
