"""A clip's results in page-locked host memory: ``InferenceCore(result_dev="cpu")``.

The reference keeps ``prob`` and ``masks`` in host RAM at ``mem_profile`` 2 and 3 (inference_core.py:44-63), so that
a clip's device footprint does not grow with its length.  Here the four host volumes of a clip — ``prob``
[(K+1), T, 1, nh, nw] fp32, the public ``masks`` [T, 1, nh, nw] u8 and the internal padded and unpadded label maps —
live in ONE pageable allocation at page-aligned offsets, page-locked in place with one ``cudaHostRegister``
(``ops.host_register``): exact size, unlike ``pin_memory()``, which rounds up to a power of two and keeps the block
cached after release.  Kernels write the volumes through the mapped device address the registration returns.

Result planes reach the volumes only through ``mivos_deliver_planes`` (``ops.deliver_planes``), which also writes
the frame's argmax into the two label maps: the label maps therefore always hold argmax(prob) of every frame ever
written, and an interaction's result is a host copy of them, not a re-read of the volume."""
from __future__ import annotations

import weakref

import torch

from . import ops

PAGE = 4096


def _page_round(n: int) -> int:
    return (n + PAGE - 1) // PAGE * PAGE


class HostResults:
    def __init__(self, k1: int, t: int, nh: int, nw: int, h: int, w: int, pad, device):
        self.k1, self.t, self.nh, self.nw, self.h, self.w = k1, t, nh, nw, h, w
        self.pad_l, self.pad_t = int(pad[0]), int(pad[2])
        plane = nh * nw
        sizes = (k1 * t * plane * 4, t * plane, t * plane, t * h * w)
        offs, total = [], 0
        for s in sizes:
            offs.append(total)
            total += _page_round(s)
        # the registered range covers whole pages of this allocation only: no page is shared with another buffer
        raw = torch.empty(total + PAGE, dtype=torch.uint8)
        skip = (-raw.data_ptr()) % PAGE
        block = raw[skip:skip + total]
        view = lambda i: block[offs[i]:offs[i] + sizes[i]]  # noqa: E731
        self.prob = view(0).view(torch.float32).view(k1, t, 1, nh, nw)
        self.masks = view(1).view(t, 1, nh, nw)
        self.labels = view(2).view(t, 1, nh, nw)
        self.labels_unpadded = view(3).view(t, h, w)
        self.fill()
        base = ops.host_register(block)
        self._finalizer = weakref.finalize(self, ops.host_unregister, block)
        self._dev_prob, self._dev_labels, self._dev_unpadded = base + offs[0], base + offs[2], base + offs[3]
        # eager deliveries (an interacted frame, a fused frame): one record, and prob[:, ti] staged on the device
        self.table = torch.zeros(ops.DELIVER_WORDS, dtype=torch.int64, device=device)
        self.frame = torch.empty((k1, 1, nh, nw), dtype=torch.float32, device=device)

    def fill(self) -> None:
        """The initial state of the reference's buffers (:77-82): prob zero but prob[0] = 1e-7, labels zero."""
        self.prob.zero_()
        self.prob[0] = 1e-7
        self.masks.zero_()
        self.labels.zero_()
        self.labels_unpadded.zero_()

    def record(self, ti: int, first_plane: int) -> list:
        """The mivos_deliver_planes record that delivers planes [first_plane, first_plane + K + 1) to frame ti."""
        plane = self.nh * self.nw
        return [self._dev_prob + ti * plane * 4, self.t * plane, self._dev_labels + ti * plane,
                self._dev_unpadded + ti * self.h * self.w, first_plane | (self.k1 << 32),
                self.pad_l | (self.pad_t << 32), self.h | (self.w << 32), 0]

    def store(self, planes: torch.Tensor, ti: int) -> None:
        """prob[:, ti] = planes [(K+1), 1, nh, nw] (device), with the frame's labels; stream-ordered."""
        ops.store_words(self.table, self.record(ti, 0))
        ops.deliver_planes(planes.contiguous(), self.table, 1, self.nh, self.nw)

    def load(self, ti: int) -> torch.Tensor:
        """prob[:, ti] on the device (non-blocking copies from the page-locked volume, one per plane)."""
        for j in range(self.k1):
            self.frame[j].copy_(self.prob[j, ti], non_blocking=True)
        return self.frame
