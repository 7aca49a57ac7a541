"""TEST INFRASTRUCTURE: PyTorch-CPU stand-ins for the per-set C-ABI operators (mivos_memory_read_sets,
mivos_bank_write_sets), written from the header's contracts on top of tests/abi_emulator.py's scalar operators.
``install`` monkeypatches them over ``mivos_b200.ops`` next to abi_emulator.install_host_runtime, so that the ragged
lock-step host loop runs on the CPU.  Nothing in the product package imports it."""
from __future__ import annotations

import torch

import abi_emulator as E


def memory_read_sets(bank_k, bank_v, slots, qk, top_k, out, counts, *, out_coff=0, halo_hw=None, workspace=None,
                     algo=0, want_topk=False):
    """Header contract of mivos_memory_read_sets: object o reads query set s = o // (k / sets) over the live slots
    0 .. counts[s] - 1 of its own bank."""
    k, sets = bank_k.shape[0], qk.shape[0]
    per = k // sets
    sel = [E.memory_read(bank_k[s * per:(s + 1) * per], bank_v[s * per:(s + 1) * per], slots, qk[s], top_k,
                         out[s * per:(s + 1) * per], out_coff=out_coff, halo_hw=halo_hw, dyn_slots=counts[s:s + 1],
                         want_topk=want_topk) for s in range(sets)]
    return (out, torch.cat([r[1] for r in sel]), torch.cat([r[2] for r in sel])) if want_topk else out


def bank_write_sets(halo, k, sets, h, w, coff_k, coff_v, bank_k, bank_v, t_max, dyn_t):
    """Header contract of mivos_bank_write_sets: set s (k / sets objects) writes bank frame dyn_t[s]; a frame
    outside [0, t_max] writes nothing."""
    per = k // sets
    for s in range(sets):
        t = int(dyn_t[s])
        if 0 <= t <= t_max:
            E.bank_write(halo[s * per:(s + 1) * per], per, h, w, coff_k, coff_v, bank_k[s * per:(s + 1) * per],
                         bank_v[s * per:(s + 1) * per], t)


OPS = ("memory_read_sets", "bank_write_sets")


def install(monkeypatch, ops_module):
    import sys
    me = sys.modules[__name__]
    for name in OPS:
        monkeypatch.setattr(ops_module, name, getattr(me, name))
