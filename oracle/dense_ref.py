"""Oracle: sentence-transformers Dense modules after Pooling, and DistilBERT's classification head, in float64.
TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

What it follows:

* sentence-transformers ``models.Dense``: ``activation_function(linear(x))`` with ``linear`` an ``nn.Linear(in_features,
  out_features, bias)``, run after ``Pooling`` and before ``Normalize`` in the module list [3P-recall: sentence-transformers
  2.6.1 is not installed here].
* transformers ``DistilBertForSequenceClassification``: ``classifier(relu(pre_classifier(h[:, 0])))``; its encoder is
  BERT's under other names and runs through ``encoder_kernels_ref.encoder_stack_ref`` with the renamed weights
  (``ragmeup_b200.weights.distilbert_to_canonical``).
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np
import torch


def _f64(a, device=None) -> torch.Tensor:
    t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    return t.to(device=device or t.device, dtype=torch.float64)


def dense_chain_ref(x, layers: Sequence[Tuple[object, Optional[object], int]], normalize: bool) -> torch.Tensor:
    """pooled rows x [B, H] -> y = act_n(W_n ... act_1(W_1 x + b_1) ... + b_n), then y / max(||y||, 1e-12) per row when
    normalize; ``layers`` as ``ragmeup_b200.weights.dense_layers`` returns them (act 0 identity, 1 tanh).  float64 on
    x's device."""
    y = _f64(x)
    for W, b, act in layers:
        y = y @ _f64(W, y.device).T
        if b is not None:
            y = y + _f64(b, y.device)[None, :]
        if int(act) == 1:
            y = torch.tanh(y)
        elif int(act) != 0:
            raise ValueError(act)
    return y / y.norm(dim=1, keepdim=True).clamp(min=1e-12) if normalize else y


def relu_head_ref(h_cls, pw, pb, cw, cb) -> torch.Tensor:
    """DistilBertForSequenceClassification's head on CLS rows [B, H]: cw relu(pw h + pb) + cb, float64"""
    h = _f64(h_cls)
    z = torch.relu(h @ _f64(pw, h.device).T + _f64(pb, h.device)[None, :])
    return z @ _f64(cw, h.device).T + _f64(cb, h.device)[None, :]
