"""Write tests/golden/generate.npz: greedy generation on tiny Llama and Qwen3 decoders with seeded weights.

    python tests/golden/make_golden_generate.py

Each model (``models()``: tiny-llama / tiny-qwen3 with a 1 024-token vocabulary, projections scaled by 6 so the top-2
margins are wide, and a seeded LM head) runs greedy generation with repetition penalty 1.2 from three prompts of 1,
9 and 40 tokens, ``STEPS`` tokens each.  Stored per (model, prompt): the prompt, the oracle's greedy tokens and the
float64 logits of the first ``LOGIT_STEPS`` steps (``oracle/generation_ref.py``).
"""
import os
import sys
from dataclasses import replace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import generation_ref as gref  # noqa: E402
from ragmeup_b200.weights import (DECODER_PRESETS, PRESETS, synthetic_llama_weights,  # noqa: E402
                                  synthetic_qwen3_weights)

KINDS = ("llama", "qwen3")
PROMPT_LENS = (1, 9, 40)
STEPS = 8
LOGIT_STEPS = 3
PENALTY = 1.2


def model(kind: str, vocab: int = 1024, scale: float = 6.0, seed: int = 3, max_pos: int = 8192):
    """(config, weights, lm_head [vocab, H]) of a tiny decoder whose vocabulary the LM head GEMM takes"""
    if kind == "llama":
        cfg = replace(DECODER_PRESETS["tiny-llama"], vocab_size=vocab, max_pos=max_pos)
        w = synthetic_llama_weights(cfg, seed=seed, scale=scale)
    else:
        cfg = replace(PRESETS["tiny-qwen3"][0], vocab_size=vocab, max_pos=max_pos, num_labels=1, reranker=False)
        w = synthetic_qwen3_weights(cfg, seed=seed, scale=scale)
    lm = (np.random.default_rng(seed + 11).standard_normal((vocab, cfg.hidden)) * 0.5).astype(np.float32)
    return cfg, w, lm


def prompts(vocab: int = 1024):
    rng = np.random.default_rng(5)
    return [rng.integers(0, vocab, T).astype(np.int32) for T in PROMPT_LENS]


def compute():
    out = {}
    for kind in KINDS:
        cfg, w, lm = model(kind)
        for i, ids in enumerate(prompts()):
            seq, toks, logits = list(ids.tolist()), [], []
            for step in range(STEPS):
                x = gref.logits(w, lm, cfg, seq, kind == "qwen3")
                if step < LOGIT_STEPS:
                    logits.append(x)
                t = gref.greedy(gref.repetition_penalty(x, seq, PENALTY))
                toks.append(t)
                seq.append(t)
            out[f"{kind}_{i}_prompt"] = ids
            out[f"{kind}_{i}_tokens"] = np.asarray(toks, np.int32)
            out[f"{kind}_{i}_logits"] = np.stack(logits)
    return out


def main() -> None:
    np.savez(os.path.join(os.path.dirname(os.path.abspath(__file__)), "generate.npz"), **compute())


if __name__ == "__main__":
    main()


CHAT_WORDS = 256
ASSISTANT = "assistant:"


def save_chat_snapshot(path: str):
    """a tiny Llama chat model as a local snapshot (config.json, model.safetensors, generation_config.json and a
    word-level tokenizer built with ``tokenizers``, no download): vocabulary 256 = <s>, </s>, <unk>, ``ASSISTANT`` and
    w4 .. w255; 2 layers, hidden 256, 2 heads over 1 kv head of 128 -> (model, tokenizer)"""
    import torch
    from tokenizers import Tokenizer, models, pre_tokenizers
    from transformers import LlamaConfig, LlamaForCausalLM, PreTrainedTokenizerFast
    vocab = {"<s>": 0, "</s>": 1, "<unk>": 2, ASSISTANT: 3}
    vocab.update({f"w{i}": i for i in range(4, CHAT_WORDS)})
    tk = Tokenizer(models.WordLevel(vocab, unk_token="<unk>"))
    tk.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    tok = PreTrainedTokenizerFast(tokenizer_object=tk, bos_token="<s>", eos_token="</s>", unk_token="<unk>")
    cfg = LlamaConfig(vocab_size=CHAT_WORDS, hidden_size=256, intermediate_size=384, num_hidden_layers=2,
                      num_attention_heads=2, num_key_value_heads=1, head_dim=128, max_position_embeddings=512,
                      rope_theta=10000.0, bos_token_id=0, eos_token_id=1, tie_word_embeddings=False,
                      initializer_range=0.2)
    torch.manual_seed(0)
    model = LlamaForCausalLM(cfg).eval()
    model.save_pretrained(path, safe_serialization=True)
    tok.save_pretrained(path)
    return model, tok
