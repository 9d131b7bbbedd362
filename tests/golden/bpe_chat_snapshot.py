"""A tiny Llama chat snapshot for the LLM provenance tests, built in-process (no download): a byte-level BPE tokenizer
trained with ``tokenizers`` on a small corpus, with a Llama-3-style chat template so ``decode(...,
skip_special_tokens=True)`` reproduces ``"assistant\\n\\n"``, and a 2-layer Llama (2 query heads over 1 kv head of
128, vocabulary 384) saved with ``save_pretrained``."""
import torch

# Jinja drops one trailing newline of a template's source: the closing empty tag keeps the header's "\n\n" whole
TEMPLATE = ("{{ bos_token }}{% for m in messages %}<|start_header_id|>{{ m['role'] }}<|end_header_id|>\n\n"
            "{{ m['content'] }}<|eot_id|>{% endfor %}<|start_header_id|>assistant<|end_header_id|>\n\n{{ '' }}")
# digits in the prompt keep the corpus (and so the vocabulary) full of number tokens, so replies often hold a number
PROMPT = "Score from 0 to 10 how well {context} supports {answer} for {query}. Reply 3, 5 or 7.5 only."


def save_bpe_chat_snapshot(path):
    """-> (model, tokenizer), both also saved under ``path``"""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers, trainers
    from transformers import LlamaConfig, LlamaForCausalLM, PreTrainedTokenizerFast
    tk = Tokenizer(models.BPE())
    tk.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tk.decoder = decoders.ByteLevel()
    special = ["<|begin_of_text|>", "<|eot_id|>", "<|start_header_id|>", "<|end_header_id|>"]
    trainer = trainers.BpeTrainer(vocab_size=384, special_tokens=special,
                                  initial_alphabet=pre_tokenizers.ByteLevel.alphabet())
    corpus = [PROMPT, "user assistant system", "the documents support answers to queries", "0 1 2 3 4 5 6 7 8 9 10"] * 20
    tk.train_from_iterator(corpus, trainer)
    tok = PreTrainedTokenizerFast(tokenizer_object=tk, bos_token="<|begin_of_text|>", eos_token="<|eot_id|>")
    tok.chat_template = TEMPLATE
    cfg = LlamaConfig(vocab_size=384, hidden_size=256, intermediate_size=384, num_hidden_layers=2,
                      num_attention_heads=2, num_key_value_heads=1, head_dim=128, max_position_embeddings=1024,
                      rope_theta=10000.0, bos_token_id=0, eos_token_id=1, tie_word_embeddings=False,
                      initializer_range=0.2)
    torch.manual_seed(0)
    model = LlamaForCausalLM(cfg).eval()
    model.save_pretrained(path, safe_serialization=True)
    tok.save_pretrained(path)
    return model, tok
