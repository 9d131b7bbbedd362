"""Host-side WordPiece tokenisation (SURVEY.md H10).

The reference tokenises with HuggingFace ``tokenizers`` (Rust) through
``BertTokenizerFast`` inside sentence-transformers (called from
``server/RAGHelper_local.py:114-117`` / ``server/RAGHelper.py:484``); it is not
GPU arithmetic and stays on the host here too, using the same library.  This
module only builds the ``tokenizers.Tokenizer`` (from a snapshot's
``tokenizer.json`` / ``vocab.txt`` or a seeded synthetic vocab) and packs
batches into the ragged ``cu_seqlens`` layout the CUDA encoder consumes
(no padding tokens are ever sent to the device).
"""
from __future__ import annotations

import functools
import os
import threading
from concurrent.futures import ThreadPoolExecutor
from itertools import chain
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
from tokenizers import Tokenizer, models, normalizers, pre_tokenizers, processors, decoders

PAD, UNK, CLS, SEP, MASK = 0, 100, 101, 102, 103

_SYL = ["ba", "ce", "di", "fo", "gu", "ha", "je", "ki", "lo", "mu", "na", "pe", "qi", "ro", "su",
        "ta", "ve", "wi", "xo", "yu", "za", "bri", "cle", "dro", "fla", "gri", "ple", "sto", "tru", "vla"]


def synthetic_vocab(size: int = 30522, seed: int = 7) -> Dict[str, int]:
    """bert-base-uncased-like id layout ([PAD]=0, [UNK]=100, [CLS]=101, [SEP]=102,
    [MASK]=103) filled with seeded pseudo-words and ##suffixes."""
    assert size >= 400
    vocab: Dict[str, int] = {}
    specials = {PAD: "[PAD]", UNK: "[UNK]", CLS: "[CLS]", SEP: "[SEP]", MASK: "[MASK]"}
    i = 0
    u = 0
    while i < 104:
        if i in specials:
            vocab[specials[i]] = i
        else:
            vocab[f"[unused{u}]"] = i
            u += 1
        i += 1
    for ch in "abcdefghijklmnopqrstuvwxyz0123456789.,;:!?'\"()-":
        vocab[ch] = i
        i += 1
    for ch in "abcdefghijklmnopqrstuvwxyz0123456789":
        vocab["##" + ch] = i
        i += 1
    rng = np.random.default_rng(seed)
    # words of up to 3 syllables give about 56 000 entries; larger vocabularies (the 105 879 of multilingual BERT)
    # take words of up to 4.  Vocabularies of BERT's usual 30 522 and smaller are unchanged.
    syllables = 4 if size > 50000 else 3
    while i < size:
        n = int(rng.integers(1, syllables + 1))
        word = "".join(_SYL[int(j)] for j in rng.integers(0, len(_SYL), n))
        if rng.random() < 0.25:
            word = "##" + word
        if word not in vocab:
            vocab[word] = i
            i += 1
    return vocab


def build_wordpiece(vocab: Dict[str, int], lowercase: bool = True) -> Tokenizer:
    tok = Tokenizer(models.WordPiece(vocab=vocab, unk_token="[UNK]", max_input_chars_per_word=100))
    tok.normalizer = normalizers.BertNormalizer(clean_text=True, handle_chinese_chars=True,
                                                strip_accents=None, lowercase=lowercase)
    tok.pre_tokenizer = pre_tokenizers.BertPreTokenizer()
    tok.post_processor = processors.TemplateProcessing(
        single="[CLS] $A [SEP]", pair="[CLS] $A [SEP] $B:1 [SEP]:1",
        special_tokens=[("[CLS]", vocab["[CLS]"]), ("[SEP]", vocab["[SEP]"])])
    tok.decoder = decoders.WordPiece(prefix="##")
    return tok


MPNET_SPECIALS = ("<s>", "<pad>", "</s>", "<unk>")    # ids 0..3; "<mask>" is the last id


def synthetic_mpnet_vocab(size: int = 30527) -> Dict[str, int]:
    """MPNet's id layout: <s>=0, <pad>=1, </s>=2, <unk>=3, then the BERT vocabulary of ``synthetic_vocab(size - 5)``
    shifted by 4 ([UNK] at 104), then <mask>."""
    vocab = {t: i for i, t in enumerate(MPNET_SPECIALS)}
    for t, i in synthetic_vocab(size - 5).items():
        vocab[t] = i + 4
    vocab["<mask>"] = size - 1
    return vocab


def build_mpnet_wordpiece(vocab: Dict[str, int]) -> Tokenizer:
    """MPNet's tokenizer: BERT normalisation and WordPiece, RoBERTa's templates ``<s> A </s>`` and
    ``<s> A </s> </s> B </s>`` (type ids 0), and the specials as added tokens, so a literal "<pad>" in a text is id 1."""
    tok = build_wordpiece(vocab)
    tok.post_processor = processors.RobertaProcessing(sep=("</s>", vocab["</s>"]), cls=("<s>", vocab["<s>"]),
                                                      trim_offsets=False, add_prefix_space=False)
    tok.add_special_tokens([*MPNET_SPECIALS, "<mask>"])
    return tok


XLMR_SPECIALS = MPNET_SPECIALS                         # <s>=0, <pad>=1, </s>=2, <unk>=3; "<mask>" is the last id
_LETTERS = "abcdefghijklmnopqrstuvwxyz0123456789.,;:!?'\"()-"


@functools.lru_cache(maxsize=4)
def synthetic_xlmr_pieces(size: int = 250002, seed: int = 11) -> Tuple[Tuple[str, float], ...]:
    """A seeded SentencePiece Unigram vocabulary of ``size`` pieces in XLM-R's id layout: the four specials, "▁", every
    letter, digit and punctuation mark with and without the "▁" word-start mark, then distinct pseudo-words of one to
    four syllables (about half of them word-initial), then <mask>.  Scores are negative log-probabilities that favour
    short pieces, so a word splits into few pieces."""
    assert size >= 400
    pieces = [(t, 0.0) for t in XLMR_SPECIALS] + [("▁", -3.0)]
    pieces += [(p + c, -8.0) for c in _LETTERS for p in ("▁", "")]
    seen = {p for p, _ in pieces}
    rng = np.random.default_rng(seed)
    need = size - 1 - len(pieces)
    while need > 0:
        m = 2 * need + 64
        n = rng.integers(1, 5, m)
        syl = rng.integers(0, len(_SYL), (m, 4))
        mark = rng.random(m) < 0.5
        score = -(n + rng.random(m))
        for k in range(m):
            w = ("▁" if mark[k] else "") + "".join(_SYL[j] for j in syl[k, :n[k]])
            if w not in seen:
                seen.add(w)
                pieces.append((w, float(score[k])))
                need -= 1
                if need == 0:
                    break
    pieces.append(("<mask>", 0.0))
    return tuple(pieces)


def build_xlmr_unigram(pieces: Sequence[Tuple[str, float]]) -> Tokenizer:
    """XLM-R's tokenizer shape: Unigram over ``pieces``, Metaspace pre-tokenisation, templates ``<s> A </s>`` and
    ``<s> A </s> </s> B </s>`` (type ids 0), and the specials as added tokens, so a literal "<pad>" is id 1."""
    tok = Tokenizer(models.Unigram(list(pieces), unk_id=3, byte_fallback=False))
    tok.pre_tokenizer = pre_tokenizers.Metaspace(replacement="▁", prepend_scheme="always")
    tok.post_processor = processors.TemplateProcessing(
        single="<s> $A </s>", pair="<s> $A </s> </s> $B </s>", special_tokens=[("<s>", 0), ("</s>", 2)])
    tok.decoder = decoders.Metaspace(replacement="▁", prepend_scheme="always")
    tok.add_special_tokens([*XLMR_SPECIALS, "<mask>"])
    return tok


DEBERTA_SPECIALS = ("[PAD]", "[CLS]", "[SEP]", "[UNK]")   # ids 0..3; "[MASK]" is the last id


def synthetic_deberta_pieces(size: int = 128100) -> Tuple[Tuple[str, float], ...]:
    """DeBERTa-v3's id layout ([PAD]=0, [CLS]=1, [SEP]=2, [UNK]=3, [MASK] last) over the pieces of
    ``synthetic_xlmr_pieces(size)``"""
    pieces = list(synthetic_xlmr_pieces(size))
    pieces[:4] = [(t, 0.0) for t in DEBERTA_SPECIALS]
    pieces[-1] = ("[MASK]", 0.0)
    return tuple(pieces)


def build_deberta_unigram(pieces: Sequence[Tuple[str, float]]) -> Tokenizer:
    """DeBERTa-v3's tokenizer shape (``DebertaV2TokenizerFast``'s tokenizer.json): Unigram over ``pieces``, Metaspace
    with ``prepend_scheme="first"``, templates ``[CLS] A [SEP]`` and ``[CLS] A [SEP] B [SEP]`` with type ids 0 / 1, and
    the specials as added tokens."""
    tok = Tokenizer(models.Unigram(list(pieces), unk_id=3, byte_fallback=False))
    tok.pre_tokenizer = pre_tokenizers.Metaspace(replacement="▁", prepend_scheme="first")
    tok.post_processor = processors.TemplateProcessing(
        single="[CLS] $A [SEP]", pair="[CLS] $A [SEP] $B:1 [SEP]:1", special_tokens=[("[CLS]", 1), ("[SEP]", 2)])
    tok.decoder = decoders.Metaspace(replacement="▁", prepend_scheme="first")
    tok.add_special_tokens([*DEBERTA_SPECIALS, "[MASK]"])
    return tok


QWEN3_SPECIALS = ("<|endoftext|>", "<|im_start|>", "<|im_end|>")


def build_byte_bpe(words: Sequence[str], specials: Sequence[str] = QWEN3_SPECIALS, append: Optional[str] = None) -> Tokenizer:
    """A byte-level BPE in Qwen's form (ByteLevel pre-tokenizer and decoder, no unknown token): the 256 byte symbols,
    then each of ``words`` (and its space-prefixed form) as one token through left-to-right merges, then ``specials`` as
    special added tokens.  ``append`` (a special): the post-processor appends it to every single text and pair, as some
    embedders' tokenizers append <|endoftext|>; else nothing is added."""
    from tokenizers import decoders, models, pre_tokenizers
    alphabet = pre_tokenizers.ByteLevel.alphabet()
    vocab = {c: i for i, c in enumerate(sorted(alphabet))}
    merges = []
    for w in words:
        for form in ("\u0120" + w, w):        # the space-prefixed form first: its merges must outrank the bare word's
            form = "".join(bytes_to_byte_level(form))
            cur = form[0]
            for ch in form[1:]:
                if cur + ch not in vocab:
                    merges.append((cur, ch))
                    vocab[cur + ch] = len(vocab)
                cur = cur + ch
    tok = Tokenizer(models.BPE(vocab=vocab, merges=merges))
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=True)
    tok.decoder = decoders.ByteLevel()
    tok.add_special_tokens(list(specials))
    if append is None:
        tok.post_processor = processors.ByteLevel(trim_offsets=False)
    else:
        tok.post_processor = processors.TemplateProcessing(single=f"$A {append}", pair=f"$A $B:1 {append}:1",
                                                           special_tokens=[(append, tok.token_to_id(append))])
    return tok


def bytes_to_byte_level(text: str) -> List[str]:
    """text -> its ByteLevel symbols (GPT-2's byte-to-unicode map; the space-prefix marker \u0120 is kept as it is)"""
    from tokenizers import pre_tokenizers
    if text.startswith("\u0120"):
        return ["\u0120"] + bytes_to_byte_level(text[1:])
    pieces = pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False).pre_tokenize_str(text)
    return list("".join(p for p, _ in pieces))


def synthetic_qwen3_tokenizer(vocab_size: int) -> Tokenizer:
    """the synthetic presets' byte-level BPE: the words of synthetic_vocab that fit below vocab_size, with the Qwen
    specials and single ``yes`` / ``no`` tokens"""
    room = max(0, vocab_size - 256 - len(QWEN3_SPECIALS) - 16)
    words = ["yes", "no"] + [w for w in synthetic_vocab(min(30522, max(room, 1))) if w.isalpha() and len(w) > 2]
    tok = build_byte_bpe(words[:max(2, room // 8)])
    if tok.get_vocab_size() > vocab_size:
        raise ValueError(f"synthetic Qwen3 tokenizer: {tok.get_vocab_size()} tokens do not fit vocab_size {vocab_size}")
    return tok


def load_tokenizer(source: Optional[str], vocab_size: int = 30522, mpnet: bool = False, xlmr: bool = False,
                   deberta: bool = False, modernbert: bool = False, qwen3: bool = False) -> Tokenizer:
    """``source`` = snapshot dir (tokenizer.json or vocab.txt) or None -> synthetic vocab; ``mpnet`` selects MPNet's
    vocabulary layout and templates where the snapshot has no tokenizer.json.  ``xlmr`` (XLM-R / RoBERTa) and
    ``deberta`` (DeBERTa-v2 / v3): a snapshot must have tokenizer.json (read by ``tokenizers``); None -> the synthetic
    Unigram vocabulary of that family.  ``modernbert``: a snapshot must have tokenizer.json (ModernBERT's BPE with the
    template ``[CLS] A [SEP] B [SEP]``); None -> the synthetic WordPiece vocabulary, which has the same template.
    ``qwen3``: a snapshot's tokenizer.json (its byte-level BPE and post-processor as they are); None -> the synthetic
    byte-level BPE of ``synthetic_qwen3_tokenizer``."""
    if qwen3:
        if source is None:
            return synthetic_qwen3_tokenizer(vocab_size)
        return Tokenizer.from_file(os.path.join(source, "tokenizer.json"))
    if modernbert and source is not None:
        tj = os.path.join(source, "tokenizer.json")
        if os.path.exists(tj):
            return Tokenizer.from_file(tj)
        raise FileNotFoundError(f"{source}: ModernBERT snapshots need tokenizer.json (its BPE tokenizer has no other "
                                f"file form)")
    if deberta:
        if source is None:
            return build_deberta_unigram(synthetic_deberta_pieces(vocab_size))
        tj = os.path.join(source, "tokenizer.json")
        if os.path.exists(tj):
            return Tokenizer.from_file(tj)
        why = (f"{source}: DeBERTa-v2 snapshots need tokenizer.json (the sentencepiece package is not a dependency; "
               f"saving the tokenizer with transformers' fast tokenizer writes it)")
        if os.path.exists(os.path.join(source, "spm.model")):
            raise ValueError(why + ", and this one has only spm.model")
        raise FileNotFoundError(why)
    if xlmr and source is None:
        return build_xlmr_unigram(synthetic_xlmr_pieces(vocab_size))
    build = build_mpnet_wordpiece if mpnet else build_wordpiece
    if source is None:
        return build(synthetic_mpnet_vocab(vocab_size) if mpnet else synthetic_vocab(vocab_size))
    tj = os.path.join(source, "tokenizer.json")
    if os.path.exists(tj):
        return Tokenizer.from_file(tj)
    if xlmr:
        why = (f"{source}: XLM-R / RoBERTa snapshots need tokenizer.json (the sentencepiece package is not a "
               f"dependency; saving the tokenizer with transformers' fast tokenizer writes it)")
        if os.path.exists(os.path.join(source, "sentencepiece.bpe.model")):
            raise ValueError(why + ", and this one has only sentencepiece.bpe.model")
        raise FileNotFoundError(why)
    vt = os.path.join(source, "vocab.txt")
    if os.path.exists(vt):
        with open(vt, encoding="utf-8") as f:
            vocab = {line.rstrip("\n"): i for i, line in enumerate(f)}
        return build(vocab)
    raise FileNotFoundError(f"{source}: neither tokenizer.json nor vocab.txt")


def synthetic_sentences(vocab: Dict[str, int], n: int, min_words: int, max_words: int, seed: int) -> List[str]:
    """Seeded pseudo-sentences made of whole vocabulary words (for tests / benches)."""
    words = [w for w in vocab if not w.startswith("[") and not w.startswith("##") and len(w) > 1]
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        k = int(rng.integers(min_words, max_words + 1))
        out.append(" ".join(words[int(j)] for j in rng.integers(0, len(words), k)))
    return out


class RaggedTokenizer:
    """A PRIVATE copy of a tokenizer, configured once (truncation='longest_first' to max_length, no
    padding) and never mutated afterwards, so any number of request threads can tokenise through it
    (Flask serves /chat on several threads over one shared RAGHelper: server/server.py:141-146,394;
    mutating a shared `tokenizers.Tokenizer` while another thread encodes raises "Already borrowed")."""

    def __init__(self, tok: Tokenizer, max_length: int):
        self.max_length = int(max_length)
        self._tok = Tokenizer.from_str(tok.to_str())
        self._tok.enable_truncation(max_length=self.max_length, strategy="longest_first")
        self._tok.no_padding()
        # single texts carry type id 0 throughout with BERT's post-processor; checked once instead of assumed
        probe = self._tok.encode("a b")
        self._single_zero = not any(probe.type_ids)

    def __call__(self, texts_a: Sequence[str], texts_b: Optional[Sequence[str]] = None):
        if texts_b is None:
            return _pack(_encode_batch(self._tok, list(texts_a)), single_segment=self._single_zero)
        return _pack(_encode_batch(self._tok, list(zip(texts_a, texts_b))))


def encode_ragged(tok: Tokenizer, texts_a: Sequence[str], texts_b: Optional[Sequence[str]],
                  max_length: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Tokenise with truncation='longest_first', NO padding, and pack (single-threaded helper: it
    re-configures `tok`; the drop-in classes use RaggedTokenizer instead).

    Returns (ids int32 [T], type_ids int32 [T], cu_seqlens int32 [B+1])."""
    tok.enable_truncation(max_length=max_length, strategy="longest_first")
    tok.no_padding()
    if texts_b is None:
        enc = _encode_batch(tok, list(texts_a))
    else:
        enc = _encode_batch(tok, list(zip(texts_a, texts_b)))
    return _pack(enc)


def _encode_batch(tok: Tokenizer, inputs, **kw):
    """``encode_batch_fast`` (tokenizers >= 0.20) skips the character-offset bookkeeping this path never reads: the same
    ids / type ids / truncation, about a third of the time on 60-word chunks — and WordPiece is what bounds bulk ingest
    and the text-level rerank.  Older wheels fall back to ``encode_batch``."""
    fast = getattr(tok, "encode_batch_fast", None)
    return fast(inputs, **kw) if fast is not None else tok.encode_batch(inputs, **kw)


def _pack(enc, single_segment: bool = False) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    id_lists = [e.ids for e in enc]                      # each .ids builds a Python list: fetch it once
    lens = np.fromiter(map(len, id_lists), dtype=np.int64, count=len(id_lists))
    cu = np.zeros(len(enc) + 1, dtype=np.int32)
    np.cumsum(lens, out=cu[1:])
    total = int(cu[-1])
    ids = np.fromiter(chain.from_iterable(id_lists), dtype=np.int32, count=total)
    if single_segment:                                   # [CLS] a [SEP]: BERT's template gives every token type 0
        typ = np.zeros(total, dtype=np.int32)
    else:
        typ = np.fromiter(chain.from_iterable(e.type_ids for e in enc), dtype=np.int32, count=total)
    return ids, typ, cu


def pipelined(chunks: Sequence, tokenize, run) -> List:
    """``[run(tokenize(c)) for c in chunks]`` with the tokenisation of chunk i+1 (host, HF `tokenizers` releases the
    GIL) overlapped with the device call of chunk i (ctypes releases the GIL while it waits on the stream): for bulk calls
    the host-side WordPiece is what is left to hide."""
    chunks = list(chunks)
    if len(chunks) <= 1:
        return [run(tokenize(c)) for c in chunks]
    out = []
    with ThreadPoolExecutor(max_workers=1) as ex:
        fut = ex.submit(tokenize, chunks[0])
        for i in range(len(chunks)):
            tok = fut.result()
            if i + 1 < len(chunks):
                fut = ex.submit(tokenize, chunks[i + 1])
            out.append(run(tok))
    return out


class PairAssembler:
    """(text_a, text_b) pairs -> the ragged batch of ``RaggedTokenizer(a, b)`` (``[CLS] a [SEP] b [SEP]`` for BERT,
    ``<s> a </s> </s> b </s>`` for XLM-R / RoBERTa), built from PER-TEXT ids that are cached.  A reranker scores the
    same documents against many queries (and the same query against many documents): with the cache only unseen texts
    reach the tokeniser.

    The special tokens around and between the two texts, and their token types, are the tokenizer's own pair template,
    read once from the post-processor's output on a probe pair.  Equality with pair tokenisation rests on two facts
    checked in tests/test_host_logic.py and tests/test_xlmr_cpu.py: normalisation and pre-tokenisation act on each
    segment separately, and `truncation="longest_first"` in HF `tokenizers` is the closed form below (shorter side n1,
    longer n2: n2 = max(n1, B - n1); if still too long n1 = B // 2, n2 = n1 + B % 2), with B = max_length minus the
    template's special tokens (three for BERT, four for RoBERTa)."""

    def __init__(self, tok: Tokenizer, max_length: int, max_entries: int = 1 << 18):
        self.max_length = int(max_length)
        self._tok = Tokenizer.from_str(tok.to_str())
        self._tok.no_truncation()
        self._tok.no_padding()
        self._pre, self._mid, self._post, self._type_a, self._type_b = self._template(self._tok)
        self._cache: Dict[str, np.ndarray] = {}
        self._max_entries = int(max_entries)
        self._lock = threading.Lock()

    @staticmethod
    def _template(tok: Tokenizer):
        """the pair template as (ids before a, ids between a and b, ids after b, type of [pre, a, mid], type of
        [b, post]) from the post-processor's output on the pair ("a", "b")"""
        e = tok.encode("a", "b")
        seq, ids, typ = e.sequence_ids, np.asarray(e.ids, dtype=np.int32), e.type_ids
        ia = [i for i, s in enumerate(seq) if s == 0]
        ib = [i for i, s in enumerate(seq) if s == 1]
        if not ia or not ib or ia != list(range(ia[0], ia[-1] + 1)) or ib != list(range(ib[0], ib[-1] + 1)) \
                or ia[-1] >= ib[0]:
            raise ValueError("PairAssembler: the tokenizer's pair template is not <specials> a <specials> b <specials>")
        a0, a1, b0, b1 = ia[0], ia[-1] + 1, ib[0], ib[-1] + 1
        if any(seq[i] is not None for i in (*range(a0), *range(a1, b0), *range(b1, len(seq)))):
            raise ValueError("PairAssembler: the pair template interleaves text and special tokens")
        ta, tb = typ[a0], typ[b0]
        if any(t != ta for t in typ[:b0]) or any(t != tb for t in typ[b0:]):
            raise ValueError("PairAssembler: the pair template's token types are not one run for a, one for b")
        return ids[:a0], ids[a1:b0], ids[b1:], int(ta), int(tb)

    def _ids(self, texts: Sequence[str]) -> List[np.ndarray]:
        got: Dict[str, np.ndarray] = {}
        with self._lock:
            for t in dict.fromkeys(texts):
                v = self._cache.get(t)
                if v is not None:
                    got[t] = v
        missing = [t for t in dict.fromkeys(texts) if t not in got]
        if missing:
            enc = _encode_batch(self._tok, missing, add_special_tokens=False)    # outside the lock: releases the GIL
            fresh = {t: np.asarray(e.ids, dtype=np.int32) for t, e in zip(missing, enc)}
            got.update(fresh)
            with self._lock:
                self._cache.update(fresh)
                while len(self._cache) > self._max_entries:                      # oldest first
                    self._cache.pop(next(iter(self._cache)))
        return [got[t] for t in texts]

    def __call__(self, texts_a: Sequence[str], texts_b: Sequence[str]) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        ia, ib = self._ids(list(texts_a)), self._ids(list(texts_b))
        la = np.fromiter(map(len, ia), dtype=np.int64, count=len(ia))
        lb = np.fromiter(map(len, ib), dtype=np.int64, count=len(ib))
        pre, mid, post = self._pre, self._mid, self._post
        budget = self.max_length - (len(pre) + len(mid) + len(post))
        swap = la > lb
        n1, n2 = np.where(swap, lb, la), np.where(swap, la, lb)
        over = la + lb > budget
        n2t = np.maximum(n1, budget - n1)
        both = n1 + n2t > budget
        n1t = np.where(both, budget // 2, n1)
        n2t = np.where(both, budget // 2 + budget % 2, n2t)
        na = np.where(over, np.where(swap, n2t, n1t), la)
        nb = np.where(over, np.where(swap, n1t, n2t), lb)
        cu = np.zeros(len(ia) + 1, dtype=np.int32)
        np.cumsum(na + nb + (len(pre) + len(mid) + len(post)), out=cu[1:])
        pieces = []
        for a, b, x, y in zip(ia, ib, na, nb):
            pieces += (pre, a[:x], mid, b[:y], post)
        ids = np.concatenate(pieces) if pieces else np.zeros(0, dtype=np.int32)
        if self._type_a == self._type_b:
            typ = np.full(int(cu[-1]), self._type_a, dtype=np.int32)
        else:                                                      # one run of type_a, then one of type_b per pair
            runs = np.stack([na + (len(pre) + len(mid)), nb + len(post)], 1).ravel()
            typ = np.repeat(np.tile(np.asarray([self._type_a, self._type_b], np.int32), len(ia)), runs)
        return ids, typ, cu
