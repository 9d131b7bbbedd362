"""NF4 blockwise quantisation as bitsandbytes applies it to the reference's chat model, restated in numpy.

``RAGHelper_local._initialize_llm`` loads the decoder with ``BitsAndBytesConfig(load_in_4bit=True,
bnb_4bit_quant_type="nf4", bnb_4bit_use_double_quant=False, bnb_4bit_compute_dtype=float16)``.  bitsandbytes cannot
run here, so every fact below about what it does is [3P-recall]: restated from bitsandbytes' ``quantize_4bit`` /
``dequantize_4bit`` (blocksize 64) and its CUDA kernels ``kQuantizeBlockwise`` / ``kDequantizeBlockwise``, and from
transformers' ``replace_with_bnb_linear``; parity with them is unverified.

* Which tensors [3P-recall]: every ``nn.Linear`` of the decoder layers (q / k / v / o, gate / up / down).  ``lm_head``
  is skipped (``llm_int8_skip_modules`` defaults to the output embedding); embeddings and norms stay unquantised.
* fp16 first [3P-recall]: ``torch_dtype`` defaults to float16 under bnb, so the bf16 checkpoint is cast to fp16
  (round to nearest even, subnormals kept) before it is quantised.
* Blocks [3P-recall]: the row-major flattened tensor in blocks of 64 consecutive elements; ``absmax`` is the fp32
  maximum of |w| over a block; each value is scaled by ``x * (1 / absmax)`` in fp32.
* Codes [3P-recall]: ``dQuantizeNF4``'s threshold tree, strict ``>`` at the midpoints of neighbouring code values.  The
  tree's answer is the number of thresholds below x, which is what ``quantize`` counts (NaN passes none: code 0).
* Packing [3P-recall]: two codes per byte, the first element in the high nibble.
* Dequantisation [3P-recall]: ``fp16(code[q] * absmax)``, the product in fp32 rounded once to fp16.
* All-zero blocks: absmax = 0 makes ``1 / absmax`` infinite and every scaled value ``0 * inf = NaN``, which passes no
  threshold: every code is 0 (-1.0) and dequantises to ``-1.0 * 0 = -0.0``, zero as the block was.

K must be a multiple of 64, so no block straddles two rows: a row re-ordering (the fused q | k | v rows, the 64 + 64
gate / up interleave of the SwiGLU rows) moves whole blocks and quantising the re-ordered weight gives the same codes.
"""
from __future__ import annotations

import numpy as np

BLOCK = 64

# Dettmers et al., QLoRA (2023), Appendix E: the 16 NF4 values, as bitsandbytes' table holds them in fp32
CODE = np.array([
    -1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635,
    -0.18477343022823334, -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725,
    0.24611230194568634, 0.33791524171829224, 0.44070982933044434, 0.5626170039176941,
    0.7229568362236023, 1.0], dtype=np.float32)

# dQuantizeNF4's thresholds in ascending order, the fp32 literals of its tree [3P-recall]
THRESHOLDS = np.array([
    -0.8480964004993439, -0.6106329262256622, -0.4599952697753906, -0.33967943489551544,
    -0.23460740596055984, -0.13791173323988914, -0.045525018125772476, 0.03979014977812767,
    0.1202552504837513, 0.2035212516784668, 0.2920137718319893, 0.3893125355243683,
    0.5016634166240692, 0.6427869200706482, 0.8614784181118011], dtype=np.float32)


def to_fp16(w) -> np.ndarray:
    """the fp16 cast the loader applies: round to nearest even, subnormals kept (numpy's float32 -> float16 cast)"""
    return np.asarray(w, dtype=np.float32).astype(np.float16)


def _check(w: np.ndarray) -> None:
    if w.ndim != 2 or w.shape[1] % BLOCK != 0:
        raise ValueError(f"NF4 weights need [N, K] with K a multiple of {BLOCK}, got shape {w.shape}")


def quantize(w16: np.ndarray):
    """fp16 [N, K] -> (packed codes uint8 [N, K / 2], absmax float32 [N, K / 64])"""
    w16 = np.asarray(w16)
    if w16.dtype != np.float16:
        raise TypeError("quantize takes the fp16 weight (to_fp16 of the checkpoint's values)")
    _check(w16)
    N, K = w16.shape
    blocks = w16.astype(np.float32).reshape(N, K // BLOCK, BLOCK)
    absmax = np.abs(blocks).max(axis=2).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = (np.float32(1.0) / absmax).astype(np.float32)
        scaled = (blocks * inv[:, :, None]).astype(np.float32)
        q = (scaled[..., None] > THRESHOLDS).sum(axis=-1).astype(np.uint8).reshape(N, K)
    packed = (q[:, 0::2] << 4) | q[:, 1::2]
    return packed.astype(np.uint8), absmax


def unpack(codes: np.ndarray) -> np.ndarray:
    """packed uint8 [N, K / 2] -> code indices uint8 [N, K] (high nibble first)"""
    codes = np.asarray(codes, dtype=np.uint8)
    q = np.empty((codes.shape[0], codes.shape[1] * 2), dtype=np.uint8)
    q[:, 0::2] = codes >> 4
    q[:, 1::2] = codes & 15
    return q


def dequantize(codes: np.ndarray, absmax: np.ndarray) -> np.ndarray:
    """(packed codes, absmax) -> fp16 [N, K] = fp16(code[q] * absmax), the product in fp32"""
    q = unpack(codes)
    N, K = q.shape
    a = np.repeat(np.asarray(absmax, dtype=np.float32), BLOCK, axis=1).reshape(N, K)
    return (CODE[q] * a).astype(np.float32).astype(np.float16)


def nf4_weight(w) -> np.ndarray:
    """a checkpoint weight as the NF4 model computes with it: fp16 cast, quantised, dequantised -> float32 [N, K]"""
    codes, absmax = quantize(to_fp16(w))
    return dequantize(codes, absmax).astype(np.float32)
