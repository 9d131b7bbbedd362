"""Device memory of the GPU decoder's generation calls: destroying a handle frees the scratch its
rmu_decoder_generate_batch calls grew, so handles that are built, used and destroyed in turn do not leak."""
from __future__ import annotations

import ctypes as C
import gc

import numpy as np
import pytest
import torch

import make_golden_generate as mg

pytestmark = pytest.mark.gpu


def _batch_cycle(cfg, w, lm, B, max_new):
    """create a handle with an LM head, run one generate_batch over B prompts, destroy the handle"""
    from ragmeup_b200 import _lib as L
    from ragmeup_b200.encoder import BertEncoder
    enc = BertEncoder(cfg, w, with_head=False)
    enc._check(L.lib().rmu_decoder_set_lm_head(enc._h, np.ascontiguousarray(lm).ctypes.data), "set_lm_head")
    prompts = [[(7 * b + 3 * t + 1) % cfg.vocab_size for t in range(4 + b)] for b in range(B)]
    ids = np.ascontiguousarray([t for p in prompts for t in p], dtype=np.int32)
    cu = np.ascontiguousarray(np.cumsum([0] + [len(p) for p in prompts]), dtype=np.int32)
    seeds = np.zeros(B, dtype=np.uint64)
    out = np.zeros((B, max_new), dtype=np.int32)
    n = np.zeros(B, dtype=np.int32)
    s = L.SamplingC(0, 1.0, 1.0, 1.0, 50, 0, (C.c_int32 * L.MAX_EOS)())
    enc._check(L.lib().rmu_decoder_generate_batch(enc._h, ids.ctypes.data, cu.ctypes.data, B, C.byref(s),
                                                  seeds.ctypes.data, max_new, out.ctypes.data, n.ctypes.data, None,
                                                  L.stream_ptr()), "rmu_decoder_generate_batch")
    assert (n == max_new).all()
    del enc
    gc.collect()
    torch.cuda.synchronize()


def test_destroy_frees_the_batch_scratch():
    """B = 16 prompts over V = 131 072: the batch's logits alone take 8 MiB, four times the driver's 2 MB granularity.
    After one cycle that loads the kernels' modules, three more create / generate_batch / destroy cycles leave the free
    device memory where it was, to the granularity of up to 2 MB for each cycle's scratch allocation."""
    cfg, w, lm = mg.model("llama", vocab=131072)
    B, max_new, cycles = 16, 2, 3
    assert B * cfg.vocab_size * 4 >= 4 * (2 << 20)
    gc.collect()
    torch.cuda.empty_cache()
    _batch_cycle(cfg, w, lm, B, max_new)
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(cycles):
        _batch_cycle(cfg, w, lm, B, max_new)
    free1 = torch.cuda.mem_get_info()[0]
    assert abs(free1 - free0) <= cycles * (2 << 20), (free0 - free1)
