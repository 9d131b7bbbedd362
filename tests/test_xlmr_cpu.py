"""CPU: XLM-RoBERTa / RoBERTa models (the bge rerankers behind HuggingFaceCrossEncoder's default, the multilingual
embedders).  The oracles against the goldens minted from transformers' XLMRobertaModel and
XLMRobertaForSequenceClassification (tests/golden/make_golden_xlmr.py); snapshot resolution from snapshots written by
transformers' own save_pretrained, and every refusal; the synthetic XLM-R tokenizer; PairAssembler against pair
tokenisation for a SentencePiece Unigram and a byte-level BPE tokenizer."""
import json
import os
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import bert_ref, xlmr_ref
from ragmeup_b200.weights import PRESETS, XLMRConfig, synthetic_bert_weights, weight_names

GOLDEN = [("bge-reranker-base", 0, 1.0, True), ("tiny-xlmr", 2, 4.0, True), ("tiny-xlmr-long", 1, 1.0, False)]


def _cfg(preset):
    return XLMRConfig(**asdict(PRESETS[preset][0]))


@pytest.mark.parametrize("preset,seed,scale,head", GOLDEN)
def test_xlmr_oracle_matches_hf(golden_dir, preset, seed, scale, head):
    """the fp32 forward (padded, pad id 1) and the float64 ragged stack both match transformers at BERT's bar, positions
    past 512 included (tiny-xlmr-long)"""
    g = np.load(f"{golden_dir}/xlmr.npz")
    key = f"xlmr_{preset}_{seed}_{scale}"
    cfg = _cfg(preset)
    ocfg = xlmr_ref.XLMRCfg(**asdict(cfg))
    w = synthetic_bert_weights(cfg, seed=seed, with_head=head, scale=scale)
    ids = torch.from_numpy(g[key + "_ids"].astype(np.int64))
    mask = torch.from_numpy(g[key + "_mask"].astype(np.int64))
    assert (ids == 1).logical_and(mask == 1).any(), "the goldens hold a literal id 1 inside a text"
    lens = mask.sum(1).tolist()
    with torch.no_grad():
        h = xlmr_ref.xlmr_encoder_forward(w, ocfg, ids, mask)
        mean = bert_ref.l2_normalize(bert_ref.pool(h, mask, "mean")).numpy()
        cls = bert_ref.l2_normalize(bert_ref.pool(h, mask, "cls")).numpy()
        logits = xlmr_ref.classifier_head(w, h).numpy() if head else None
    h_last = np.stack([h[b, n - 1].numpy() for b, n in enumerate(lens)])
    tol = 4e-6 if scale == 1.0 else 2e-5
    assert np.abs(mean - g[key + "_mean"]).max() < tol
    assert np.abs(cls - g[key + "_cls"]).max() < tol
    assert np.abs(h[:, 0].numpy() - g[key + "_h_first"]).max() < 50 * tol
    assert np.abs(h_last - g[key + "_h_last"]).max() < 50 * tol
    if head:
        want = g[key + "_logits"]
        assert np.abs(logits - want).max() < 50 * tol * max(1.0, float(np.abs(want).max()))
    # the float64 reference of the kernels, on the ragged batch
    flat = np.concatenate([g[key + "_ids"][b, :n] for b, n in enumerate(lens)])
    cu = np.r_[0, np.cumsum(lens)]
    ref = xlmr_ref.xlmr_stack_ref(w, cfg, flat, cu)
    assert float((ref["mean_norm"] - torch.from_numpy(g[key + "_mean"]).double()).abs().max()) < tol
    assert float((ref["cls_norm"] - torch.from_numpy(g[key + "_cls"]).double()).abs().max()) < tol
    assert float((ref["hidden"][cu[1:] - 1] - torch.from_numpy(g[key + "_h_last"]).double()).abs().max()) < 50 * tol
    if head:
        want = torch.from_numpy(g[key + "_logits"]).double()
        assert float((ref["logits"] - want).abs().max()) < 50 * tol * max(1.0, float(want.abs().max()))


# ------------------------------------------------------------------------------------------ snapshots and refusals
def _hc(cfg, **kw):
    from transformers import XLMRobertaConfig
    return XLMRobertaConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden, num_hidden_layers=cfg.layers,
                            num_attention_heads=cfg.heads, intermediate_size=cfg.ffn,
                            max_position_embeddings=cfg.max_pos, type_vocab_size=1, layer_norm_eps=1e-5, pad_token_id=1,
                            **kw)


def _save(model, path, safe=True, tokenizer=True, model_max_length=None, patch=None):
    model.save_pretrained(path)
    if not safe:                  # the older format alone (transformers 5 writes safetensors whatever it is asked)
        os.remove(os.path.join(path, "model.safetensors"))
        torch.save(model.state_dict(), os.path.join(path, "pytorch_model.bin"))
    if tokenizer:
        from ragmeup_b200.tokenizer import load_tokenizer
        load_tokenizer(None, model.config.vocab_size, xlmr=True).save(os.path.join(path, "tokenizer.json"))
    if model_max_length is not None:
        with open(os.path.join(path, "tokenizer_config.json"), "w") as f:
            json.dump({"model_max_length": model_max_length}, f)
    if patch:
        with open(os.path.join(path, "config.json")) as f:
            conf = json.load(f)
        conf.update(patch)
        with open(os.path.join(path, "config.json"), "w") as f:
            json.dump(conf, f)
    return path


def _canonical(sd, head):
    """the model's own tensors under the canonical names (the test's independent statement of the mapping)"""
    out = {}
    for k, v in sd.items():
        k = k.replace("roberta.", "", 1)
        if k.startswith("classifier.dense."):
            k = "pooler.dense." + k[len("classifier.dense."):]
        elif k.startswith("classifier.out_proj."):
            k = "classifier." + k[len("classifier.out_proj."):]
        elif k.startswith("pooler.") and not head:
            continue
        out[k] = v.detach().numpy()
    return out


@pytest.mark.parametrize("safe", [True, False])                    # model.safetensors, or pytorch_model.bin only
def test_cross_encoder_snapshot_from_save_pretrained(tmp_path, safe):
    from transformers import XLMRobertaForSequenceClassification
    from ragmeup_b200.tokenizer import load_tokenizer
    from ragmeup_b200.weights import resolve_model
    cfg = _cfg("tiny-xlmr")
    torch.manual_seed(0)
    m = XLMRobertaForSequenceClassification(_hc(cfg, num_labels=1)).eval()
    path = _save(m, str(tmp_path / "bge-reranker-base"), safe=safe, model_max_length=100)
    assert os.path.exists(os.path.join(path, "model.safetensors" if safe else "pytorch_model.bin"))
    got_cfg, w, _pool, _norm, max_len, act, src = resolve_model(path, with_head=True)
    assert isinstance(got_cfg, XLMRConfig) and (got_cfg.position_mode, got_cfg.rel_buckets, got_cfg.type_vocab) == (1, 0, 1)
    assert (got_cfg.ln_eps, got_cfg.num_labels, max_len, act, src) == (1e-5, 1, 100, "sigmoid", path)
    want = _canonical(m.state_dict(), True)
    for name, shape in weight_names(got_cfg, True):
        assert w[name].shape == shape and np.array_equal(w[name], want[name]), name
    assert w["embeddings.token_type_embeddings.weight"].any()          # the trained row, not zeroed
    # the model's own logits equal the oracle's on the resolved weights (the head mapping, end to end)
    ids = torch.tensor([[0, 17, 1, 99, 2, 2, 5, 6, 2], [0, 33, 2, 2, 44, 2, 1, 1, 1]])
    mask = torch.tensor([[1] * 9, [1] * 6 + [0] * 3])
    with torch.no_grad():
        want_logits = m(input_ids=ids, attention_mask=mask).logits
        got_logits = xlmr_ref.classifier_head(w, xlmr_ref.xlmr_encoder_forward(w, xlmr_ref.XLMRCfg(**asdict(got_cfg)),
                                                                                 ids, mask))
    assert float((got_logits - want_logits).abs().max()) < 1e-5
    # truncation: min(model_max_length, max_pos - 2)
    _save(m, path, safe=safe, tokenizer=False, model_max_length=10 ** 30)
    assert resolve_model(path, with_head=True)[4] == cfg.max_pos - 2
    os.remove(os.path.join(path, "tokenizer_config.json"))
    assert resolve_model(path, with_head=True)[4] == cfg.max_pos - 2
    assert load_tokenizer(path, cfg.vocab_size, xlmr=True).token_to_id("<pad>") == 1


def test_embedder_snapshot_with_sentence_transformers_modules(tmp_path):
    from transformers import XLMRobertaModel
    from ragmeup_b200.weights import resolve_model
    cfg = _cfg("tiny-xlmr")
    torch.manual_seed(1)
    m = XLMRobertaModel(_hc(cfg)).eval()                              # with its pooler, which an embedder ignores
    path = _save(m, str(tmp_path / "bge-m3"), model_max_length=8192)
    os.makedirs(os.path.join(path, "1_Pooling"))
    with open(os.path.join(path, "modules.json"), "w") as f:
        json.dump([{"path": "", "type": "sentence_transformers.models.Transformer"},
                   {"path": "1_Pooling", "type": "sentence_transformers.models.Pooling"},
                   {"path": "2_Normalize", "type": "sentence_transformers.models.Normalize"}], f)
    with open(os.path.join(path, "1_Pooling", "config.json"), "w") as f:
        json.dump({"pooling_mode_cls_token": True, "pooling_mode_mean_tokens": False}, f)
    with open(os.path.join(path, "sentence_bert_config.json"), "w") as f:
        json.dump({"max_seq_length": 96}, f)
    got_cfg, w, pooling, normalize, max_len, act, _src = resolve_model(path, with_head=False)
    assert isinstance(got_cfg, XLMRConfig) and (pooling, normalize, max_len, act) == ("cls", True, 96, "identity")
    want = _canonical(m.state_dict(), False)
    for name, shape in weight_names(got_cfg, False):
        assert np.array_equal(w[name], want[name]), name
    assert not any(k.startswith("pooler.") for k in w)
    # the bare pooler never stands in for a classification head
    with pytest.raises(KeyError, match="classifier"):
        resolve_model(path, with_head=True)
    # a RoBERTa model_type reads the same way
    _save(m, path, tokenizer=False, patch={"model_type": "roberta"})
    assert isinstance(resolve_model(path, with_head=False)[0], XLMRConfig)


@pytest.mark.parametrize("patch,match", [
    ({"pad_token_id": 0}, "pad_token_id"),
    ({"position_embedding_type": "relative_key"}, "absolute position"),
    ({"hidden_act": "gelu_new"}, "erf-GELU"),
    ({"model_type": "camembert"}, "camembert"),
    ({"model_type": "distilbert"}, "distilbert"),
    ({"model_type": "electra"}, "electra"),
])
def test_config_refusals(tmp_path, patch, match):
    """each refused before any weight is read; an unprefixed camembert snapshot (BERT's tensor names) used to load as
    BERT, with BERT's positions"""
    from transformers import XLMRobertaModel
    from ragmeup_b200.weights import resolve_model
    m = XLMRobertaModel(_hc(_cfg("tiny-xlmr")), add_pooling_layer=False)
    path = _save(m, str(tmp_path / "m"), tokenizer=False, patch=patch)
    with pytest.raises(ValueError, match=match):
        resolve_model(path, with_head=False)


def test_tokenizer_and_flashrank_refusals(tmp_path):
    from transformers import XLMRobertaForSequenceClassification
    from ragmeup_b200.flashrank import Ranker
    from ragmeup_b200.tokenizer import load_tokenizer
    from ragmeup_b200.weights import resolve_model
    cfg = _cfg("tiny-xlmr")
    m = XLMRobertaForSequenceClassification(_hc(cfg, num_labels=1))
    # only sentencepiece.bpe.model: refused, naming tokenizer.json
    path = _save(m, str(tmp_path / "sp"), tokenizer=False)
    open(os.path.join(path, "sentencepiece.bpe.model"), "wb").close()
    src = resolve_model(path, with_head=True)[6]
    with pytest.raises(ValueError, match="tokenizer.json"):
        load_tokenizer(src, cfg.vocab_size, xlmr=True)
    os.remove(os.path.join(path, "sentencepiece.bpe.model"))
    with pytest.raises(FileNotFoundError, match="tokenizer.json"):
        load_tokenizer(src, cfg.vocab_size, xlmr=True)
    # an XLM-R snapshot under a FlashRank name, and an XLM-R preset, are not FlashRank models
    _save(m, str(tmp_path / "ms-marco-MiniLM-L-12-v2"))
    for make in (lambda: Ranker("ms-marco-MiniLM-L-12-v2", cache_dir=str(tmp_path)),
                 lambda: Ranker("synthetic:tiny-xlmr")):
        with pytest.raises(ValueError, match="XLM-R"):
            make()


def test_presets():
    from ragmeup_b200.weights import resolve_model
    shapes = {"bge-reranker-base": (250002, 768, 12, 12, 3072, 514, "cls", True, 512),
              "bge-reranker-v2-m3": (250002, 1024, 24, 16, 4096, 8194, "cls", True, 8192),
              "multilingual-e5-small": (250037, 384, 12, 12, 1536, 514, "mean", True, 512),
              "multilingual-e5-base": (250002, 768, 12, 12, 3072, 514, "mean", True, 512),
              "bge-m3": (250002, 1024, 24, 16, 4096, 8194, "cls", True, 8192),
              "paraphrase-multilingual-mpnet-base-v2": (250002, 768, 12, 12, 3072, 514, "mean", False, 128)}
    for name, want in shapes.items():
        c, pooling, max_len = PRESETS[name]
        assert isinstance(c, XLMRConfig) and c.head_dim in (32, 64)
        norm = resolve_model(f"synthetic:{name}", with_head=False)[3] if name == "multilingual-e5-small" else \
            name != "paraphrase-multilingual-mpnet-base-v2"
        assert (c.vocab_size, c.hidden, c.layers, c.heads, c.ffn, c.max_pos, pooling, norm, max_len) == want, name
    assert _cfg("tiny-xlmr").head_dim == 32 and _cfg("tiny-xlmr-long").max_pos == 8194
    r = resolve_model("synthetic:tiny-xlmr", with_head=True)
    assert r[5] == "sigmoid" and r[1]["embeddings.token_type_embeddings.weight"].any()
    assert resolve_model("synthetic:tiny-xlmr-long", with_head=False)[3:5] == (True, 8192)


# ------------------------------------------------------------------------------------------------------ tokenizers
def test_synthetic_xlmr_tokenizer():
    from ragmeup_b200.tokenizer import RaggedTokenizer, load_tokenizer, synthetic_xlmr_pieces
    tok = load_tokenizer(None, 2000, xlmr=True)
    pieces = synthetic_xlmr_pieces(2000)
    assert len(pieces) == 2000 == tok.get_vocab_size() and len({p for p, _ in pieces}) == 2000
    assert [tok.token_to_id(t) for t in ("<s>", "<pad>", "</s>", "<unk>", "<mask>")] == [0, 1, 2, 3, 1999]
    assert synthetic_xlmr_pieces(2000) == synthetic_xlmr_pieces(2000, 11)        # seeded
    e = tok.encode("ba ce")
    assert e.ids[0] == 0 and e.ids[-1] == 2 and 3 not in e.ids and not any(e.type_ids)
    p = tok.encode("ba", "ce")
    ba, ce = tok.token_to_id("▁ba"), tok.token_to_id("▁ce")
    assert p.ids == [0, ba, 2, 2, ce, 2] and not any(p.type_ids)
    e = tok.encode("ba <pad> ce <mask>")                  # literal specials are the special tokens, attention mask 1
    assert 1 in e.ids and 1999 in e.ids and e.attention_mask == [1] * len(e.ids)
    ids, typ, cu = RaggedTokenizer(tok, 4)(["<pad>", "ba ce di fo"])
    assert ids[:3].tolist() == [0, 1, 2] and cu.tolist() == [0, 3, 7] and not typ.any()


def _bpe_tokenizer():
    """a byte-level BPE tokenizer with RoBERTa's post-processor, trained here on seeded text"""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers, processors, trainers
    tok = Tokenizer(models.BPE())
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tok.decoder = decoders.ByteLevel()
    rng = np.random.default_rng(0)
    syl = ["ba", "ce", "di", "fo", "gu", "ha", "je", "ki", "lo", "mu"]
    corpus = [" ".join("".join(rng.choice(syl, rng.integers(1, 4))) for _ in range(20)) for _ in range(300)]
    tok.train_from_iterator(corpus, trainers.BpeTrainer(vocab_size=700, show_progress=False,
                                                        special_tokens=["<s>", "<pad>", "</s>", "<unk>", "<mask>"],
                                                        initial_alphabet=pre_tokenizers.ByteLevel.alphabet()))
    tok.post_processor = processors.RobertaProcessing(sep=("</s>", 2), cls=("<s>", 0), trim_offsets=True,
                                                      add_prefix_space=False)
    return tok


def _one_piece_words(tok, cands):
    enc = tok.encode_batch(cands, add_special_tokens=False)
    return [w for w, e in zip(cands, enc) if len(e.ids) == 1]


@pytest.mark.parametrize("kind", ["unigram", "bpe"])
def test_pair_assembler_equals_pair_tokenisation(kind):
    """every (len_a, len_b) around the four-token budget of max_length, empty texts, literal <pad> / <mask>, cache
    eviction, and seeded texts of many lengths"""
    from ragmeup_b200.tokenizer import PairAssembler, RaggedTokenizer, load_tokenizer
    if kind == "unigram":
        tok = load_tokenizer(None, 2000, xlmr=True)
        words = _one_piece_words(tok, sorted(p[1:] for p in tok.get_vocab() if p.startswith("▁") and len(p) > 2))
    else:
        tok = _bpe_tokenizer()
        words = _one_piece_words(tok, ["ba", "ce", "di", "fo", "gu", "ha", "je", "ki", "lo", "mu"])
        words = [w for w in words if len(_one_piece_words(tok, [" " + w])) == 1]
    assert len(words) >= 8
    pre, mid, post, ta, tb = PairAssembler._template(tok)
    assert (pre.tolist(), mid.tolist(), post.tolist(), ta, tb) == ([0], [2, 2], [2], 0, 0)
    rng = np.random.default_rng(3)
    text = lambda n: " ".join(rng.choice(words, n)) if n else ""    # noqa: E731  n pieces (each word one piece)
    for max_length in (4, 5, 6, 7, 8, 9, 12):
        a, b = [], []
        for la in range(0, max_length + 3):
            for lb in range(0, max_length + 3):
                a.append(text(la))
                b.append(text(lb))
        a += ["<pad>", "x <mask> y", "", "<pad> <pad>"]
        b += ["<mask>", "", "<pad>", text(3)]
        rt, pa = RaggedTokenizer(tok, max_length), PairAssembler(tok, max_length, max_entries=16)
        for got, want in zip(pa(a, b), rt(a, b)):
            assert np.array_equal(got, want), max_length
        for got, want in zip(pa(a[::-1], b[::-1]), rt(a[::-1], b[::-1])):      # after evictions
            assert np.array_equal(got, want), max_length
        assert len(pa._cache) <= 16
    # the budget is max_length - 4: a pair of 2 + 2 pieces fits 8 and is cut to 1 + 2 at 7
    pa = PairAssembler(tok, 7)
    two_a, two_b = text(2), text(2)
    assert np.diff(pa([two_a], [two_b])[2]).tolist() == [7]
    assert np.diff(PairAssembler(tok, 8)([two_a], [two_b])[2]).tolist() == [8]
    long = [text(int(n)) for n in rng.integers(0, 300, 40)]
    for max_length in (64, 128, 512):
        rt, pa = RaggedTokenizer(tok, max_length), PairAssembler(tok, max_length)
        for got, want in zip(pa(long, long[::-1]), rt(long, long[::-1])):
            assert np.array_equal(got, want), max_length
