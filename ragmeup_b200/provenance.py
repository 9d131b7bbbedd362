"""Provenance attribution helpers that reuse the encoder / cross-encoder / cosine primitives (SURVEY.md §8 row f4).

Drop-ins for the four attribution methods of ``server/provenance.py`` that sit on this path:

* ``compute_attention`` (``server/provenance.py:19-98``): how much last-layer attention the query and the answer
  exchange with each retrieved document inside the chat thread, from a Llama or Qwen3 decoder on the GPU
  (``DecoderAttention``).  The decoder sums the softmax over token spans directly; no attention map is stored.

* ``compute_llm_provenance`` (``server/provenance.py:110-141``): ask the chat decoder to score each document for the
  answer, one scoring prompt per document, every prompt decoded in one batched call (``generate_batch``).

* ``compute_rerank_provenance`` (``server/provenance.py:100-108``): re-score the retrieved documents against
  ``answer`` (or ``query + "\\n" + answer`` when ``attribute_include_query == "True"``) with the reranker.
* ``DocumentSimilarityAttribution.compute_similarity`` (``server/provenance.py:164-202``): sentence-embed answer,
  query and documents, cosine of every document with the answer (and the query), average, normalise by the sum.

The reference's ``SentenceTransformer.encode`` + sklearn ``cosine_similarity`` become ``HuggingFaceEmbeddings``
(BERT on the GPU) + one brute-force cosine search over the documents (``FlatIndex``); nothing runs on the CPU but
the final handful of float32 additions.
"""
from __future__ import annotations

import ctypes as C
import logging
import os
import re
import threading
from typing import Any, List, Optional, Sequence

import numpy as np

from . import _lib, decode_session
from .index import FlatIndex
from .weights import (GB, check_decoder_plan, decoder_config, decoder_layers, decoder_lm_head, find_snapshot,
                      resolve_decoder)


def compute_rerank_provenance(reranker: Any, query: str, documents: Sequence[Any], answer: str) -> Sequence[Any]:
    if os.getenv("attribute_include_query") == "True":
        full_text = query + "\n" + answer
    else:
        full_text = answer
    # same document list back, each with metadata["relevance_score"] (ScoredCrossEncoderReranker)
    return reranker.compress_documents(documents, full_text)


class DocumentSimilarityAttribution:
    def __init__(self, model_name: Optional[str] = None, embeddings: Any = None):
        if os.getenv("force_cpu") == "True":
            raise _lib.RmuError("force_cpu=True: ragmeup_b200 runs on CUDA (sm_90a) only")
        if embeddings is None:
            from .embeddings import HuggingFaceEmbeddings
            embeddings = HuggingFaceEmbeddings(model_name=model_name or os.getenv("provenance_similarity_llm"),
                                               model_kwargs={"device": "cuda"})
        self.model = embeddings

    def compute_similarity(self, query: str, context: Sequence[Any], answer: str) -> List[float]:
        include_query = os.getenv("attribute_include_query") != "False"
        texts = [c.page_content if hasattr(c, "page_content") else str(c) for c in context]
        n = len(texts)
        if n == 0:
            return []
        # SentenceTransformer.encode only strips; encode_tensor also maps "\n" to " " (langchain's embed_documents),
        # which the BERT normaliser (clean_text) does to every whitespace character anyway: same tokens
        enc = self.model.encode_tensor
        ctx = enc(texts)
        probes = enc([answer, query] if include_query else [answer])
        idx = FlatIndex(int(ctx.shape[1]), "cosine", device=ctx.device.index)
        idx.add(ctx)
        scores, ids = idx.search(probes, n)                   # every document, sorted by similarity
        scores, ids = scores.cpu().numpy(), ids.cpu().numpy()
        sim = np.zeros((probes.shape[0], n), dtype=np.float32)
        for r in range(probes.shape[0]):
            sim[r, ids[r]] = scores[r]
        if include_query:
            similarity = [(sim[0, i] + sim[1, i]) / 2 for i in range(n)]
        else:
            similarity = [sim[0, i] for i in range(n)]
        total = sum(similarity)
        out = [s / total for s in similarity] if total > 0 else similarity
        return [float(s) for s in out]


class DecoderAttention:
    """A Llama or Qwen3 decoder (``weights.resolve_decoder``: a snapshot directory or ``synthetic:<preset>``) on the
    GPU, for attention provenance and text generation (``llms.HuggingFacePipeline``).  Its weights are uploaded once;
    ``span_mass`` then runs one thread per call, and ``generate`` attaches the LM head the first time it runs.

    ``weights="nf4"`` builds the handle in NF4 one layer at a time (``weights.decoder_layers``,
    ``BertEncoder.nf4_decoder``), as the reference's bitsandbytes load holds the model: host memory holds the embeddings
    and one layer, the device the finished handle and one staging chunk, and hidden sizes up to 8192 (the 70B class)
    load.  ``"split"`` keeps the fp32-accurate split planes, up to hidden 4096.  The device-memory plan
    (``weights.decoder_memory_plan``) is checked from the config before any tensor is read: split weights above hidden
    4096, and an NF4 plan larger than the device's free memory, raise ValueError naming the bytes and the setting."""

    def __init__(self, model_name: str, device: Optional[int] = None, weights: str = "split"):
        from .encoder import BertEncoder
        if weights not in DECODER_WEIGHTS:
            raise ValueError(f"DecoderAttention: weights must be one of {DECODER_WEIGHTS}, got {weights!r}")
        cfg = decoder_config(model_name)
        check_decoder_plan(cfg, weights)
        torch = _lib.require_cuda()
        dev = torch.cuda.current_device() if device is None else device
        # split handles build as they always did; the NF4 build, whose size the plan states exactly, is refused when
        # it cannot fit
        self.plan = check_decoder_plan(cfg, weights, torch.cuda.mem_get_info(dev)[0] if weights == "nf4" else None)
        self.model_name = model_name
        self.weights = weights
        if weights == "nf4":
            layers = decoder_layers(model_name)
            self.cfg = layers.cfg
            self.encoder = BertEncoder.nf4_decoder(layers, device=dev)
            del layers
        else:
            cfg, w = resolve_decoder(model_name)
            self.cfg = cfg
            self.encoder = BertEncoder(cfg, w, with_head=False, device=dev)
            del w
        self.lock = threading.Lock()
        self._lm_head = False
        self._scheduler = None

    @property
    def name(self) -> str:
        return self.cfg.name

    def span_mass(self, ids: Sequence[int], spans: Sequence[Sequence[int]]) -> np.ndarray:
        """the last layer's attention summed over heads, the rows of span a and the keys of span b -> float64
        [n, n]; spans are [start, end) token ranges of ``ids`` (``rmu_decoder_attention_spans``)"""
        T = len(ids)
        if T > self.cfg.max_pos:
            raise ValueError(f"{self.name}: a thread of {T} tokens exceeds max_position_embeddings ({self.cfg.max_pos})")
        if T == 0 or len(spans) == 0:
            raise ValueError(f"{self.name}: attention provenance needs a non-empty thread and at least one span")
        enc = self.encoder
        torch = enc.torch
        d_ids = enc._dev(np.asarray(ids, dtype=np.int32), torch.int32)
        d_spans = enc._dev(np.asarray(spans, dtype=np.int32).reshape(-1, 2), torch.int32)
        out = torch.empty((len(spans), len(spans)), dtype=torch.float64, device=enc.device)
        with torch.cuda.device(enc.device):
            enc._check(_lib.lib().rmu_decoder_attention_spans(enc._h, d_ids.data_ptr(), T, d_spans.data_ptr(), len(spans),
                                                              out.data_ptr(), _lib.stream_ptr()),
                       "rmu_decoder_attention_spans")
        return out.cpu().numpy()


    def generate(self, ids: Sequence[int], max_new_tokens: int, do_sample: bool = False, temperature: float = 1.0,
                 top_k: int = 50, top_p: float = 1.0, repetition_penalty: float = 1.0, eos_token_ids=(),
                 seed: int = 0, prompt_lookup_num_tokens: int = 0, max_matching_ngram_size: int = 2,
                 assistant: Optional["DecoderAttention"] = None, num_assistant_tokens: int = 20,
                 num_assistant_tokens_schedule: str = "constant") -> List[int]:
        """the new token ids after the prompt ``ids`` (``rmu_decoder_generate``'s tokens), the eos token included when
        one ends the run.  Concurrent calls share the handle's decode session (``decode_session``): a call joins it at
        the next step boundary, so a second caller's reply starts before the first one's ends, and each reply is bit for
        bit its solo run.  ``prompt_lookup_num_tokens`` > 0 drafts that many tokens (at most 15) per pass from earlier
        matches of the last ``max_matching_ngram_size``-gram (``rmu_decoder_generate_lookup``, one whole call): the
        same tokens, bit for bit, in fewer model passes when the reply copies the prompt.  ``assistant``, another
        DecoderAttention sharing this one's vocabulary, drafts ``num_assistant_tokens`` tokens (at most 15) per pass
        with its own model, the count moving per pass with ``num_assistant_tokens_schedule`` ``"heuristic"`` or
        ``"heuristic_transient"`` (``rmu_decoder_generate_assisted``, one whole call): the same tokens again, bit for
        bit, whatever the draft computes."""
        if assistant is not None and prompt_lookup_num_tokens:
            raise ValueError(f"{self.name}: prompt_lookup_num_tokens and assistant are both set: one drafter per reply")
        if max_new_tokens < 1:
            return []
        s = self._sampling(do_sample, temperature, top_k, top_p, repetition_penalty, eos_token_ids)
        enc = self.encoder
        if assistant is not None:
            return self._generate_assisted(ids, s, seed, max_new_tokens, assistant, num_assistant_tokens,
                                           num_assistant_tokens_schedule)
        if not prompt_lookup_num_tokens:
            req = decode_session.Request(ids, s, seed, max_new_tokens, name=self.name)
            with enc.torch.cuda.device(enc.device):
                try:
                    return list(self.scheduler().run(req))
                except decode_session.SessionBusy as e:
                    raise _lib.RmuError(f"rmu_decoder_generate failed: {e}") from e
        prompt = np.ascontiguousarray(list(ids), dtype=np.int32)
        out = np.zeros(int(max_new_tokens), dtype=np.int32)
        n = C.c_int32(0)
        with self.lock, enc.torch.cuda.device(enc.device):
            self._attach_lm_head()
            enc._check(_lib.lib().rmu_decoder_generate_lookup(
                enc._h, prompt.ctypes.data, len(prompt), C.byref(s), int(seed) & (2 ** 64 - 1), int(max_new_tokens),
                int(prompt_lookup_num_tokens), int(max_matching_ngram_size), out.ctypes.data, C.byref(n), None, None,
                _lib.stream_ptr()), "rmu_decoder_generate_lookup")
        return out[:n.value].tolist()

    def _generate_assisted(self, ids, s, seed, max_new_tokens, assistant, num_tokens, schedule) -> List[int]:
        """``generate`` with the draft model ``assistant``: each LM head is attached under its own handle's lock, then
        the C call (which holds both handles) runs under neither Python lock, so two calls with swapped roles cannot
        deadlock"""
        if not isinstance(assistant, DecoderAttention):
            raise ValueError(f"{self.name}: assistant must be a DecoderAttention, got {type(assistant).__name__}")
        if assistant is self:
            raise ValueError(f"{self.name}: assistant is the target's own decoder: the draft must be another handle")
        if schedule not in ASSIST_SCHEDULES:
            raise ValueError(f"{self.name}: num_assistant_tokens_schedule must be one of {tuple(ASSIST_SCHEDULES)}, "
                             f"got {schedule!r}")
        for dec in (self, assistant):
            with dec.lock, dec.encoder.torch.cuda.device(dec.encoder.device):
                dec._attach_lm_head()
        enc = self.encoder
        prompt = np.ascontiguousarray(list(ids), dtype=np.int32)
        out = np.zeros(int(max_new_tokens), dtype=np.int32)
        n = C.c_int32(0)
        with enc.torch.cuda.device(enc.device):
            enc._check(_lib.lib().rmu_decoder_generate_assisted(
                enc._h, assistant.encoder._h, prompt.ctypes.data, len(prompt), C.byref(s), int(seed) & (2 ** 64 - 1),
                int(max_new_tokens), int(num_tokens), ASSIST_SCHEDULES[schedule], out.ctypes.data, C.byref(n), None,
                None, None, None, _lib.stream_ptr()), "rmu_decoder_generate_assisted")
        return out[:n.value].tolist()

    def _sampling(self, do_sample, temperature, top_k, top_p, repetition_penalty, eos_token_ids) -> "_lib.SamplingC":
        """the C sampling settings of ``generate`` and ``generate_batch``; more than ``_lib.MAX_EOS`` eos ids raise"""
        eos = [int(t) for t in eos_token_ids]
        if len(eos) > _lib.MAX_EOS:
            raise ValueError(f"{self.name}: at most {_lib.MAX_EOS} eos ids, got {len(eos)}")
        return _lib.SamplingC(int(bool(do_sample)), float(temperature), float(top_p), float(repetition_penalty),
                              int(top_k or 0), len(eos), (C.c_int32 * _lib.MAX_EOS)(*eos))

    def _attach_lm_head(self) -> None:
        """``rmu_decoder_set_lm_head`` the first time it is needed (under ``self.lock``)"""
        if not self._lm_head:
            enc = self.encoder
            W = decoder_lm_head(self.model_name, self.cfg)
            enc._check(_lib.lib().rmu_decoder_set_lm_head(enc._h, W.ctypes.data), "rmu_decoder_set_lm_head")
            self._lm_head = True

    def scheduler(self) -> "decode_session.Scheduler":
        """the handle's decode session and its caller-driven scheduler, made (with the LM head) on first use"""
        if self._scheduler is not None:
            return self._scheduler
        with self.lock:
            if self._scheduler is None:
                with self.encoder.torch.cuda.device(self.encoder.device):
                    self._attach_lm_head()
                    self._scheduler = decode_session.Scheduler(decode_session.DecodeSession(self.encoder))
            return self._scheduler

    def generate_batch(self, prompts: Sequence[Sequence[int]], max_new_tokens: int, seeds: Sequence[int],
                       do_sample: bool = False, temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0,
                       repetition_penalty: float = 1.0, eos_token_ids=()) -> List[List[int]]:
        """``generate`` on every prompt with its own seed, in calls of up to ``_lib.MAX_GENERATE_BATCH`` prompts
        (``rmu_decoder_generate_batch``: their common prefix is prefilled once and the decode steps run all live rows
        together).  Entry b is bit for bit ``generate(prompts[b], max_new_tokens, seed=seeds[b], ...)``."""
        if len(seeds) != len(prompts):
            raise ValueError(f"{self.name}: one seed per prompt, got {len(seeds)} for {len(prompts)} prompts")
        if max_new_tokens < 1 or len(prompts) == 0:
            return [[] for _ in prompts]
        s = self._sampling(do_sample, temperature, top_k, top_p, repetition_penalty, eos_token_ids)
        enc = self.encoder
        result: List[List[int]] = []
        with self.lock, enc.torch.cuda.device(enc.device):
            self._attach_lm_head()
            for b0 in range(0, len(prompts), _lib.MAX_GENERATE_BATCH):
                part = [list(p) for p in prompts[b0:b0 + _lib.MAX_GENERATE_BATCH]]
                B = len(part)
                ids = np.ascontiguousarray([t for p in part for t in p], dtype=np.int32)
                cu = np.ascontiguousarray(np.cumsum([0] + [len(p) for p in part]), dtype=np.int32)
                sd = np.ascontiguousarray([int(x) & (2 ** 64 - 1) for x in seeds[b0:b0 + B]], dtype=np.uint64)
                out = np.zeros((B, int(max_new_tokens)), dtype=np.int32)
                n = np.zeros(B, dtype=np.int32)
                enc._check(_lib.lib().rmu_decoder_generate_batch(enc._h, ids.ctypes.data, cu.ctypes.data, B, C.byref(s),
                                                                 sd.ctypes.data, int(max_new_tokens), out.ctypes.data,
                                                                 n.ctypes.data, None, _lib.stream_ptr()),
                           "rmu_decoder_generate_batch")
                result += [out[b, :n[b]].tolist() for b in range(B)]
        return result


# transformers' num_assistant_tokens_schedule -> rmu_decoder_generate_assisted's schedule; both heuristics move k
# within one call (the assistant's config is not updated)
ASSIST_SCHEDULES = {"constant": 0, "heuristic": 1, "heuristic_transient": 1}

DECODER_WEIGHTS = ("split", "nf4")
DECODER_WEIGHTS_ENV = "RMU_DECODER_WEIGHTS"


def decoder_weights() -> str:
    """the weights a decoder handle gets: ``$RMU_DECODER_WEIGHTS`` (``split`` or ``nf4``), ``split`` when unset, so
    the reference's ``.env`` can select NF4 as its own ``BitsAndBytesConfig`` does"""
    v = os.environ.get(DECODER_WEIGHTS_ENV, "split").strip().lower() or "split"
    if v not in DECODER_WEIGHTS:
        raise ValueError(f"{DECODER_WEIGHTS_ENV}={os.environ[DECODER_WEIGHTS_ENV]!r}: expected one of {DECODER_WEIGHTS}")
    return v


# one decoder per (snapshot, device, weights): compute_attention and llms.HuggingFacePipeline share its weights.  The
# lock makes the first lookup build it once when several threads ask at the same time (each build uploads the model).
_DECODERS: dict = {}
_DECODERS_LOCK = threading.Lock()


def _decoder(model: Any) -> DecoderAttention:
    """``model`` as compute_attention takes it: a DecoderAttention, a model name, or a transformers model whose
    ``name_or_path`` names a snapshot (found as every other drop-in finds one); one handle per (path, device,
    ``decoder_weights()``)"""
    if isinstance(model, DecoderAttention):
        return model
    name = model if isinstance(model, str) else getattr(model, "name_or_path", None)
    if not name:
        raise TypeError("compute_attention: model must be a DecoderAttention, a model name or a transformers model with "
                        "name_or_path")
    weights = decoder_weights()
    torch = _lib.require_cuda()
    key = (name if name.startswith("synthetic:") else os.path.realpath(find_snapshot(name)), torch.cuda.current_device(),
           weights)
    with _DECODERS_LOCK:
        if key not in _DECODERS:
            if not isinstance(model, str):
                # the plan's refusals (split weights above hidden 4096) come before the model is touched
                plan = check_decoder_plan(decoder_config(name), weights)
                release_model_if_needed(model, plan["build_peak"], key[1], weights)
            _DECODERS[key] = DecoderAttention(name, device=key[1], weights=weights)
        return _DECODERS[key]


log = logging.getLogger(__name__)


def _cuda_tensors(model: Any, device: int):
    """the model's parameters and buffers on CUDA device ``device``"""
    for m in model.modules():
        for table in (m._parameters, m._buffers):
            for t in table.values():
                if t is not None and t.is_cuda and t.device.index == device:
                    yield t


def _held_bytes(t) -> int:
    """a tensor's bytes, with bitsandbytes' absmax when it is on CUDA"""
    import torch
    n = t.numel() * t.element_size()
    absmax = getattr(getattr(t, "quant_state", None), "absmax", None)
    if isinstance(absmax, torch.Tensor) and absmax.is_cuda:
        n += absmax.numel() * absmax.element_size()
    return n


def release_model_if_needed(model: Any, need: int, device: int, weights: str = "") -> int:
    """The reference keeps its transformers copy of the chat model loaded (``RAGHelper_local._initialize_llm``, NF4 via
    bitsandbytes), and the drop-ins read only its ``name_or_path``, ``config`` and ``generation_config``.  When the
    decoder's planned ``need`` bytes do not fit in the device's free memory beside that copy, but do fit once the copy's
    CUDA parameters and buffers on ``device`` are freed, free them (each becomes an empty CPU tensor, bitsandbytes'
    quantisation state dropped), return the cached blocks to the driver (``torch.cuda.empty_cache``: the decoder
    allocates with cudaMalloc, outside torch's allocator) and log the bytes released.  The model keeps its attributes
    but can no longer run a forward.  When even that would not make room, raise ValueError naming the bytes and leave
    the model as it was.  Returns the bytes released (0 when the decoder fits and nothing changes)."""
    import torch
    if getattr(model, "modules", None) is None:
        return 0
    free = torch.cuda.mem_get_info(device)[0]
    if need <= free:
        return 0
    held = sum(_held_bytes(t) for t in _cuda_tensors(model, device))
    if need > free + held:
        raise ValueError(
            f"{getattr(model, 'name_or_path', 'model')}: the GPU decoder needs {need} bytes ({need / GB:.1f} GB) with "
            f"RMU_DECODER_WEIGHTS={weights or 'split'}; the device has {free} bytes free and the transformers model "
            f"holds {held} bytes on it, so freeing the model would not make room: the model is left as it was")
    freed = 0
    for t in list(_cuda_tensors(model, device)):
        freed += _held_bytes(t)
        t.data = torch.empty(0, dtype=t.dtype)
        if getattr(t, "quant_state", None) is not None:
            t.quant_state = None
    torch.cuda.empty_cache()
    log.warning("released %d bytes (%.1f GB) of %s's CUDA parameters and buffers: the GPU decoder needs %d bytes and "
                "did not fit beside them; the transformers model can no longer run forwards", freed, freed / GB,
                getattr(model, "name_or_path", "the model"), need)
    return freed


def _find_part(thread: List[int], part: List[int]):
    """the first occurrence of ``part`` in ``thread`` as the reference slices it, [i : i + len - 1] (its last token
    left out; an empty part is [0 : -1]), normalised as Python normalises that slice -> [start, end)"""
    n = len(part)
    for i in range(len(thread) - n + 1):
        if thread[i:i + n] == part:
            s, e, _ = slice(i, i + n - 1).indices(len(thread))
            return s, max(s, e)
    raise ValueError("Sublist not found")


def compute_attention(model: Any, tokenizer: Any, thread: str, query: str, context: Sequence[Any],
                      answer: str) -> List[np.float64]:
    """each document's share of the attention the query and answer exchange with the documents and each other in the
    last layer, over the mean of all those shares (the reference's return value: one np.float64 per document)"""
    include_query = os.getenv("attribute_include_query") != "False"
    dec = _decoder(model)

    def enc(text):
        return list(tokenizer.encode(text, add_special_tokens=False))

    ids = enc(thread)
    texts = [c.page_content if hasattr(c, "page_content") else c for c in context]
    spans = [_find_part(ids, enc(query)), _find_part(ids, enc(answer))] + [_find_part(ids, enc(t)) for t in texts]
    mass = dec.span_mass(ids, spans)
    heads = dec.cfg.heads

    def mean(x, y):
        n = heads * (spans[x][1] - spans[x][0]) * (spans[y][1] - spans[y][0])
        return mass[x, y] / n if n else np.float64("nan")

    Q, A = 0, 1
    total = [v for v in (mean(Q, Q), mean(Q, A), mean(A, A), mean(A, Q)) if v > 0]
    scores = []
    for d in range(2, len(spans)):
        pairs = [(A, d), (d, A)] + ([(Q, d), (d, Q)] if include_query else [])
        kept = [v for v in (mean(x, y) for x, y in pairs) if v > 0]
        total += kept
        scores.append(np.mean(kept) if kept else np.float64("nan"))
    mean_total = np.mean(total) if total else np.float64("nan")
    return [np.float64(sc / mean_total) for sc in scores]


def _llm_prompt(tokenizer: Any, query: str, doc: Any, answer: str) -> List[int]:
    """the scoring prompt's ids for one document, as the reference builds it: ``provenance_llm_prompt`` formatted with
    the query, the document and the answer, as the one user message of the chat template, tokenised by the caller's
    tokenizer with truncation (and the special tokens it adds).  A ``Document`` gets its page_content's braces doubled
    in place and is formatted through ``str``, as the reference does; a ``str`` is the document's text."""
    if isinstance(doc, str):
        text = doc
    else:
        doc.page_content = doc.page_content.replace("{", "{{").replace("}", "}}")
        text = str(doc)
    prompt = os.environ["provenance_llm_prompt"].format_map({"query": query, "context": text, "answer": answer})
    chat = tokenizer.apply_chat_template([{"role": "user", "content": prompt}], tokenize=False)
    return list(tokenizer(chat, truncation=True)["input_ids"])


def _llm_score(tokenizer: Any, ids: Sequence[int], new: Sequence[int]) -> str:
    """the reference's parse of one reply: the decoded thread after its last ``assistant\n\n`` (ValueError when
    absent), commas as decimal points, the last number in it (IndexError when there is none)"""
    text = tokenizer.decode(list(ids) + list(new), skip_special_tokens=True)
    reply = text[text.rindex("assistant\n\n") + len("assistant\n\n"):]
    return re.findall(r"\d+\.?\d*", reply.replace(",", "."))[-1]


def compute_llm_provenance(tokenizer: Any, model: Any, query: str, context: Sequence[Any], answer: str) -> List[str]:
    """each document's score as the chat decoder states it (the reference's return value: one string per document).
    ``model`` resolves through ``_decoder``, so the handle is the one ``compute_attention`` and
    ``llms.HuggingFacePipeline`` use; the settings are ``model.generation_config`` with ``max_new_tokens=10``, refused
    as the pipeline refuses them; the seeds are drawn from torch's CPU default generator, one per document in order.
    Every document is scored against ``answer`` (INTEGRATION.md lists where this differs from the reference)."""
    import torch
    from .llms import resolve_settings
    if os.getenv("force_cpu") == "True":
        raise _lib.RmuError("force_cpu=True: ragmeup_b200 runs on CUDA (sm_90a) only")
    dec = _decoder(model)
    tokenizer.pad_token = tokenizer.eos_token
    tokenizer.pad_token_id = tokenizer.convert_tokens_to_ids(tokenizer.pad_token)
    tokenizer.eos_token_id = tokenizer.convert_tokens_to_ids(tokenizer.eos_token)
    prompts = [_llm_prompt(tokenizer, query, doc, answer) for doc in context]
    if not prompts:
        return []
    settings = resolve_settings(getattr(model, "generation_config", None), {"max_new_tokens": 10},
                                max(len(p) for p in prompts))
    max_new = settings.pop("max_new_tokens")
    settings.pop("prompt_lookup_num_tokens", None)     # the batched path does not draft; its tokens are the same
    settings.pop("max_matching_ngram_size", None)
    for key in ("assistant_model", "num_assistant_tokens", "num_assistant_tokens_schedule"):
        settings.pop(key, None)
    seeds = [int(torch.randint(0, 2 ** 63 - 1, (1,)).item()) for _ in prompts]
    new = dec.generate_batch(prompts, max_new, seeds, **settings)
    return [_llm_score(tokenizer, p, n) for p, n in zip(prompts, new)]
