"""mivos_b200 — Blackwell-native space-time-memory mask propagation behind the MiVOS call surface.

Public surface (mirrors the reference's import paths through the top-level shim modules
``inference_core``, ``model.propagation.prop_net``, ``model.fusion_net``, ``model.aggregate``,
``util.tensor_util``):
    InferenceCore, PropagationNetwork, FusionNet, aggregate_wbg, aggregate_sbg,
    pad_divide_by, unpad, unpad_3dim
Everything computes through ``libmivos_b200.so`` (hand-written sm_90a CUDA behind the C ABI in
include/mivos_b200.h).  There is no CPU or PyTorch fallback: ops raise if the library is missing
or the device is not an H100.
"""
from .aggregate import aggregate_sbg, aggregate_wbg  # noqa: F401
from .attn_network import AttentionReadNetwork  # noqa: F401
from .fusion_net import FusionNet  # noqa: F401
from .inference_core import InferenceCore  # noqa: F401
from .lockstep import LockstepSession  # noqa: F401
from .prop_net import PropagationNetwork  # noqa: F401
from .s2m import S2MController, S2MNetwork  # noqa: F401
from .tensor_util import pad_divide_by, unpad, unpad_3dim  # noqa: F401

__all__ = ["InferenceCore", "LockstepSession", "PropagationNetwork", "FusionNet", "AttentionReadNetwork", "S2MNetwork", "S2MController", "aggregate_wbg", "aggregate_sbg", "pad_divide_by",
           "unpad", "unpad_3dim"]
