"""TEST INFRASTRUCTURE: PyTorch-CPU stand-ins for the host-result entry points (mivos_deliver_planes,
mivos_host_register / _unregister), written from the header's contracts.  ``install`` monkeypatches them over
``mivos_b200.ops`` next to abi_emulator.install_host_runtime, so that InferenceCore(result_dev="cpu") and lock-step
sessions with host results run on the CPU.  The "device address" of a CPU tensor is its address.  Nothing in the
product package imports it."""
from __future__ import annotations

import ctypes

import torch

DELIVERED = []  # (clips) of every deliver_planes call, for the tests that count them


def _at(addr: int, n: int, dtype) -> torch.Tensor:
    size = torch.empty((), dtype=dtype).element_size()
    return torch.frombuffer((ctypes.c_uint8 * (n * size)).from_address(addr), dtype=dtype, count=n)


def deliver_planes(planes, table, clips, nh, nw):
    """Record c of `table`: planes[first : first + K+1] to the volume at word 0 (plane stride word 1), their argmax
    (first maximum) to the padded labels at word 2 and, unpadded, to word 3; a null volume or a plane count outside
    1..256 skips the clip."""
    DELIVERED.append(clips)
    plane = nh * nw
    flat = planes.reshape(-1, plane)
    for c in range(clips):
        r = [int(v) for v in table[c * 8:(c + 1) * 8]]
        first, k1 = r[4] & 0xFFFFFFFF, r[4] >> 32
        pad_l, pad_t, h, w = r[5] & 0xFFFFFFFF, r[5] >> 32, r[6] & 0xFFFFFFFF, r[6] >> 32
        if r[0] == 0 or not 1 <= k1 <= 256:
            continue
        src = flat[first:first + k1]
        for j in range(k1):
            _at(r[0] + j * r[1] * 4, plane, torch.float32).copy_(src[j])
        lab = torch.argmax(src, dim=0).to(torch.uint8)
        _at(r[2], plane, torch.uint8).copy_(lab)
        _at(r[3], h * w, torch.uint8).copy_(lab.view(nh, nw)[pad_t:pad_t + h, pad_l:pad_l + w].reshape(-1))


def host_register(t):
    return t.data_ptr()


def host_unregister(t):
    pass


OPS = ("deliver_planes", "host_register", "host_unregister")


def install(monkeypatch, ops_module):
    import sys
    me = sys.modules[__name__]
    DELIVERED.clear()
    for name in OPS:
        monkeypatch.setattr(ops_module, name, getattr(me, name))
