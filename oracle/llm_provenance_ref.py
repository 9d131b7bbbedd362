"""LLM provenance (``provenance_method=llm``) restated for the tests: each document's scoring prompt, the settings and
the reply's parse as the reference's ``compute_llm_provenance`` has them, with each reply generated one document at a
time by ``generation_ref.generate`` in float64.  Every document is scored against the caller's ``answer``, and a
``str`` document is its own text (INTEGRATION.md lists both deviations)."""
from __future__ import annotations

import os
import re
from typing import Any, List, Sequence

from . import generation_ref as gref

END = "assistant\n\n"


def prompt_ids(tokenizer: Any, query: str, doc: Any, answer: str) -> List[int]:
    if isinstance(doc, str):
        content = doc
    else:
        doc.page_content = doc.page_content.replace("{", "{{").replace("}", "}}")
        content = doc
    text = os.getenv("provenance_llm_prompt").format_map({"query": query, "context": content, "answer": answer})
    chat = tokenizer.apply_chat_template([{"role": "user", "content": text}], tokenize=False)
    return list(tokenizer(chat, truncation=True)["input_ids"])


def parse(tokenizer: Any, ids: Sequence[int], new: Sequence[int]) -> str:
    text = tokenizer.decode(list(ids) + list(new), skip_special_tokens=True)
    reply = text[text.rindex(END) + len(END):]
    return re.findall(r"\d+\.?\d*", reply.replace(",", "."))[-1]


def compute(tokenizer: Any, w, lm_head, cfg, qk_norm: bool, query: str, context: Sequence[Any], answer: str,
            settings: dict, seeds: Sequence[int]) -> List[str]:
    """``settings``: ``llms.resolve_settings``'s dict (max_new_tokens 10 for the reference's call)"""
    out = []
    for doc, seed in zip(context, seeds):
        ids = prompt_ids(tokenizer, query, doc, answer)
        new = gref.generate(w, lm_head, cfg, ids, settings["max_new_tokens"], qk_norm, do_sample=settings["do_sample"],
                            temp=settings["temperature"], k=settings["top_k"], p=settings["top_p"],
                            penalty=settings["repetition_penalty"], eos=settings["eos_token_ids"], seed=seed)
        out.append(parse(tokenizer, ids, new))
    return out
