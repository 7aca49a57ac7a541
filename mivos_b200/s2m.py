"""Drop-in Scribble-to-Mask network and controller (SURVEY.md §8f-3) — the step right before the
propagation path in both callers of the reference.

Reference surface kept:
  * ``model.s2m.s2m_network.deeplabv3plus_resnet50(num_classes=1, output_stride=16,
    pretrained_backbone=False)`` (model/s2m/s2m_network.py:55-65) -> a module with the reference's
    368-tensor ``state_dict`` (``backbone.*`` / ``classifier.*``), ``.cuda() .eval() .to()
    .load_state_dict()``, and ``net(inputs[n,6,H,W]) -> logits[n,1,H,W]`` (model/s2m/utils.py:16-21)
  * ``interact.s2m_controller.S2MController(s2m_net, num_objects, ignore_class, device)`` with
    ``interact(image, prev_mask, scr_mask) -> [K,1,nh,nw]`` (interact/s2m_controller.py:10-37)

The network runs on the same wgmma implicit-GEMM convolution as the propagation path
(engine.S2MEngine); there is no CPU or PyTorch path.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import arch
from . import _lib
from ._lib import MivosError
from .engine import S2MEngine
from .tensor_util import pad_divide_by


class S2MNetwork(nn.Module):
    def __init__(self, num_classes: int = 1, output_stride: int = 16, pretrained_backbone: bool = False,
                 act_dtype: Optional[torch.dtype] = None):
        super().__init__()
        if num_classes != 1 or output_stride != 16:
            raise MivosError("S2MNetwork: only the configuration the reference uses (num_classes=1, output_stride=16) is built")
        if pretrained_backbone:
            raise MivosError("S2MNetwork: pretrained_backbone needs a download (s2m_resnet.py:166-169); load a checkpoint instead")
        self.act_dtype = act_dtype
        arch.build_param_tree(self, arch.s2m_entries(), torch.Generator().manual_seed(2))
        self._engine: Optional[S2MEngine] = None
        self.eval()

    def _sig(self):
        return tuple((t.data_ptr(), t.dtype, t.device) for t in list(self.parameters()) + list(self.buffers()))

    def _apply(self, fn, *a, **k):
        before = self._sig()
        r = super()._apply(fn, *a, **k)
        if self._sig() != before:  # a no-op .to(device) (davis_processor.py:17) keeps the packed weights
            self._engine = None
        return r

    def load_state_dict(self, *a, **k):
        self._engine = None
        return super().load_state_dict(*a, **k)

    def engine(self) -> S2MEngine:
        p = next(self.parameters())
        _lib.require_cuda_device(p.device, "S2MNetwork")
        if self._engine is None or self._engine.device != p.device:
            sd = {k: v.detach().float() for k, v in self.state_dict().items()}
            self._engine = S2MEngine(sd, p.device, act_dtype=self.act_dtype)
        return self._engine

    @staticmethod
    def _prep(x: torch.Tensor) -> torch.Tensor:
        if x.dim() != 4 or x.shape[1] != 6:
            raise MivosError(f"S2M input must be [n,6,H,W] (image, previous mask, +/- scribbles), got {tuple(x.shape)}")
        if x.shape[-2] % 16 or x.shape[-1] % 16:
            raise MivosError("S2M input must be padded to multiples of 16 (pad_divide_by), as both reference callers do")
        return x.detach().float().contiguous()

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """logits [n,1,H,W] (callers apply torch.sigmoid: davis_processor.py:68, s2m_controller.py:35)."""
        return self.engine().forward(self._prep(x), sigmoid=False)

    def forward_sigmoid(self, x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """sigmoid(forward(x)) with the sigmoid fused into the final resize kernel."""
        return self.engine().forward(self._prep(x), sigmoid=True, out=out)


def deeplabv3plus_resnet50(num_classes: int = 1, output_stride: int = 16, pretrained_backbone: bool = False) -> S2MNetwork:
    """model/s2m/s2m_network.py:55-65."""
    return S2MNetwork(num_classes, output_stride, pretrained_backbone)


def scribble_inputs(image: torch.Tensor, prev_mask: torch.Tensor, pos: np.ndarray, neg: np.ndarray) -> torch.Tensor:
    """The 6-channel S2M inputs of ALL objects of an interaction as one batch [K,6,nh,nw]:
    cat(image, prev_mask == ki, pad(Rs_ki)) for ki = 1..K (s2m_controller.py:28-34,
    davis_processor.py:57-66).  image [1,3,nh,nw] (padded, on the device), prev_mask [1,nh,nw] label
    map, pos / neg: bool/uint8 arrays [K,h,w] (unpadded scribble maps of each object)."""
    k = pos.shape[0]
    dev = image.device
    rs = torch.from_numpy(np.stack([pos, neg], 1).astype(np.float32)).to(dev)  # [K,2,h,w]
    rs, _ = pad_divide_by(rs, 16, rs.shape[-2:])
    nh, nw = image.shape[-2:]
    x = torch.empty((k, 6, nh, nw), dtype=torch.float32, device=dev)
    x[:, 0:3] = image.float()
    labels = torch.arange(1, k + 1, device=dev, dtype=prev_mask.dtype).view(k, 1, 1)
    x[:, 3] = (prev_mask.to(dev).view(1, nh, nw) == labels).float()
    x[:, 4:6] = rs
    return x


class S2MController:
    """interact/s2m_controller.py:10-37.  With an ``S2MNetwork`` the K per-object forward passes of the
    reference loop run as ONE batch of K through the engine (sigmoid fused into the last kernel); any
    other callable network is called once per object, as the reference loop does."""

    def __init__(self, s2m_net, num_objects: int, ignore_class: int, device="cuda:0"):
        self.s2m_net = s2m_net
        self.num_objects = num_objects
        self.ignore_class = ignore_class
        self.device = device

    def interact(self, image: torch.Tensor, prev_mask: torch.Tensor, scr_mask: np.ndarray) -> torch.Tensor:
        image = image.to(self.device, non_blocking=True)
        prev_mask = prev_mask.to(self.device, non_blocking=True)
        ids = np.arange(1, self.num_objects + 1).reshape(-1, 1, 1)
        pos = scr_mask[None] == ids
        neg = (scr_mask[None] != ids) & (scr_mask[None] != self.ignore_class)
        x = scribble_inputs(image, prev_mask, pos, neg)
        if isinstance(self.s2m_net, S2MNetwork):
            return self.s2m_net.forward_sigmoid(x)
        return torch.cat([torch.sigmoid(self.s2m_net(x[i:i + 1])) for i in range(self.num_objects)], 0)
