"""Drop-in ``AttentionReadNetwork`` (reference: model/attn_network.py:30-80) — SURVEY.md §8(f) row 2.

The batch-B, two-object, training-time twin of ``PropagationNetwork.get_attention``: FusionNet
training (model/fusion_model.py:81-85) calls it under no_grad for every batch to turn the two
objects' mask differences into attention maps.  Same sub-module names as the propagation network
(``mask_rgb_encoder / rgb_encoder / kv_m_f16 / kv_q_f16``), so
``load_state_dict(prop_checkpoint, strict=False)`` keeps working (fusion_model.py:187).

Runs on the kernels of the propagation path: the 5-channel memory encoder with K = 2 objects
(each object's "other" mask is the second object's mask, attn_network.py:60-61), the query encoder,
and mivos_attention_map (softmax over the memory axis, area pooling, row-vector product, bilinear
resize; mivos_attention_map_streamed above 6912 key pixels) — W [HW, HW] is never written to memory.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch import nn

from . import arch, ops
from . import _lib
from ._lib import MivosError
from .engine import PropagationEngine


class AttentionReadNetwork(nn.Module):
    def __init__(self, act_dtype: Optional[torch.dtype] = None):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        arch.build_param_tree(self, arch.attention_read_entries(), g)
        for p in self.parameters():  # attn_network.py:40-41
            p.requires_grad = False
        self.act_dtype = act_dtype
        self._engine: Optional[PropagationEngine] = None
        self.eval()

    def _tensor_signature(self):
        return tuple((t.data_ptr(), t.dtype, t.device) for t in list(self.parameters()) + list(self.buffers()))

    def _apply(self, fn, *a, **k):
        before = self._tensor_signature()
        r = super()._apply(fn, *a, **k)
        if self._tensor_signature() != before:
            self._engine = None
        return r

    def load_state_dict(self, *a, **k):
        self._engine = None
        return super().load_state_dict(*a, **k)

    def engine(self) -> PropagationEngine:
        p = next(self.parameters())
        _lib.require_cuda_device(p.device, "AttentionReadNetwork")
        if self._engine is None:
            sd = {k: v.detach().float() for k, v in self.state_dict().items()}
            self._engine = PropagationEngine(sd, p.device, top_k=50, act_dtype=self.act_dtype)
        return self._engine

    @staticmethod
    def _f32(t: torch.Tensor) -> torch.Tensor:
        return t.detach().float().contiguous()

    @torch.no_grad()
    def forward(self, image, mask11, mask21, mask12, mask22, query_image) -> Tuple[torch.Tensor, torch.Tensor]:
        """attn_network.py:48-80: image, query_image [b,3,H,W]; masks [b,1,H,W] -> two [b,2,H,W] maps."""
        eng = self.engine()
        image, query_image = self._f32(image), self._f32(query_image)
        m11, m21, m12, m22 = (self._f32(m) for m in (mask11, mask21, mask12, mask22))
        b, _, H, W = m11.shape
        if H % 16 or W % 16:
            raise MivosError("AttentionReadNetwork: H and W must be multiples of 16 (the reference's encoders assume it)")
        h, w = H // 16, W // 16
        pos1, neg1 = (m21 - m11).clamp(0, 1), (m11 - m21).clamp(0, 1)  # :54-57
        pos2, neg2 = (m22 - m12).clamp(0, 1), (m12 - m22).clamp(0, 1)
        out1 = torch.empty((b, 2, H, W), dtype=torch.float32, device=image.device)
        out2 = torch.empty_like(out1)
        mk = torch.empty((2, h * w, 128), dtype=torch.float32, device=image.device)
        qs = None
        attention_map = ops.attention_op(h * w)
        for i in range(b):
            # objects (mask21, other = mask22) and (mask22, other = mask21): one K = 2 memory pass (:59-60)
            kv = eng.encode_memory(image[i:i + 1], torch.cat([m21[i:i + 1], m22[i:i + 1]], 0))
            ops.halo_to_pixels(kv, 2, h, w, 0, 128, mk)
            qs = eng.encode_query(query_image[i:i + 1], qs)  # :62-63
            out1[i:i + 1] = attention_map(mk[0], qs.qk, h, w, pos1[i:i + 1].contiguous(), neg1[i:i + 1].contiguous())
            out2[i:i + 1] = attention_map(mk[1], qs.qk, h, w, pos2[i:i + 1].contiguous(), neg2[i:i + 1].contiguous())
        return out1, out2
