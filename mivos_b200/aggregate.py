"""Drop-in soft aggregation (reference: model/aggregate.py).  CUDA tensors only."""
from __future__ import annotations

import torch

from . import ops


def aggregate_wbg(prob: torch.Tensor, keep_bg: bool = False, hard: bool = False) -> torch.Tensor:
    """aggregate.py:22-37: bg = prod(1-p); clamp; logit (x1000 if hard); softmax over K+1.  1 <= K <= 255."""
    return ops.aggregate_any(prob.detach().float().contiguous(), keep_bg=keep_bg, hard=hard)


def aggregate_sbg(prob: torch.Tensor, keep_bg: bool = False, hard: bool = False) -> torch.Tensor:
    """aggregate.py:4-20: constant 0.5 background instead of prod(1-p).  1 <= K <= 255."""
    return ops.aggregate_any(prob.detach().float().contiguous(), keep_bg=keep_bg, hard=hard, const_bg=True)


def aggregate_wbg_channel(prob: torch.Tensor, keep_bg: bool = False, hard: bool = False):
    """aggregate.py:39-54 — the channel-axis, autograd-carrying twin used only by FusionNet TRAINING
    (model/fusion_model.py:10,87).  Training is outside the propagation hot path (SURVEY.md §8, "out of
    scope"): this is a plain differentiable PyTorch statement so that ``import model.fusion_model``
    resolves through the shim packages; it launches no kernel of this library."""
    import torch.nn.functional as F
    new_prob = torch.cat([torch.prod(1 - prob, dim=1, keepdim=True), prob], 1).clamp(1e-7, 1 - 1e-7)
    logits = torch.log(new_prob / (1 - new_prob))
    if hard:
        logits = logits * 1000
    sm = F.softmax(logits, dim=1)
    return (logits, sm) if keep_bg else (logits, sm[:, 1:])
