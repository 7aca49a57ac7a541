"""TEST INFRASTRUCTURE: PyTorch-CPU stand-ins for the object-group C-ABI operators (mivos_*_groups), written from the
header's contracts on top of tests/abi_emulator.py's operators.  ``install`` monkeypatches them over
``mivos_b200.ops`` next to abi_emulator.install_host_runtime, so that a mixed-object lock-step session runs on the
CPU.  Nothing in the product package imports it."""
from __future__ import annotations

import torch

import abi_emulator as E


def _ranges(first):
    f = [int(v) for v in first]
    return [(f[g], f[g + 1]) for g in range(len(f) - 1)]


def memory_read_groups(bank_k, bank_v, slots, qk, top_k, out, counts, first, *, out_coff=0, halo_hw=None,
                       workspace=None, algo=0, want_topk=False):
    """Object o of group g (first[g] <= o < first[g+1]) reads query set g over the live slots 0 .. counts[g] - 1."""
    sel = [E.memory_read(bank_k[a:b], bank_v[a:b], slots, qk[g], top_k, out[a:b], out_coff=out_coff, halo_hw=halo_hw,
                         dyn_slots=counts[g:g + 1], want_topk=want_topk) for g, (a, b) in enumerate(_ranges(first))]
    return (out, torch.cat([r[1] for r in sel]), torch.cat([r[2] for r in sel])) if want_topk else out


def bank_write_groups(halo, n, h, w, coff_k, coff_v, bank_k, bank_v, t_max, dyn_t, first):
    """Group g writes its maps into bank frame dyn_t[g]; a frame outside [0, t_max] writes nothing."""
    for g, (a, b) in enumerate(_ranges(first)):
        t = int(dyn_t[g])
        if 0 <= t <= t_max:
            E.bank_write(halo[a:b], b - a, h, w, coff_k, coff_v, bank_k[a:b], bank_v[a:b], t)


def stem_gather_groups(frames, planes, n, first, out):
    """Map i, object i - first[g] of group g: frame g and the group's object planes first[g] + g + 1 + j; "others"
    sums over group g only."""
    H, W = frames.shape[-2:]
    rows = (H // 2 + 2) * (W // 2 + 2)
    for g, (a, b) in enumerate(_ranges(first)):
        E.stem_gather(frames[g:g + 1], planes[a + g + 1:b + g + 1], out[a * rows:b * rows], s2d=True)
    return out


def upsample2x_add_groups(x, up, n, h, w, skip, first, x_relu=None):
    for g, (a, b) in enumerate(_ranges(first)):
        E.upsample2x_add(x[a:b], up[a:b], b - a, h, w, x_relu=None if x_relu is None else x_relu[a:b],
                         skip=skip[g:g + 1])
    return x


def halo_copy_groups(src, dst, n, h, w, c, first, *, src_coff=0, dst_coff=0, relu=False):
    for g, (a, b) in enumerate(_ranges(first)):
        E.halo_copy(src[g:g + 1], dst[a:b], b - a, h, w, c, src_coff=src_coff, dst_coff=dst_coff, relu=relu)
    return dst


def upsample4x_sigmoid_aggregate_groups(logits, n, h4, w4, first, coff=0, raw_out=None, prob_out=None):
    """Within each group: upsample, sigmoid, aggregate_wbg(keep_bg=True) into the packed planes (group g's
    background at first[g] + g, then its objects)."""
    for g, (a, b) in enumerate(_ranges(first)):
        E.upsample4x_sigmoid_aggregate(logits[a:b], b - a, h4, w4, coff,
                                       raw_out=None if raw_out is None else raw_out[a:b],
                                       prob_out=prob_out[a + g:b + g + 1], want_raw=raw_out is not None)
    return raw_out, prob_out


OPS = ("memory_read_groups", "bank_write_groups", "stem_gather_groups", "upsample2x_add_groups", "halo_copy_groups",
       "upsample4x_sigmoid_aggregate_groups")


def install(monkeypatch, ops_module):
    import sys
    me = sys.modules[__name__]
    for name in OPS:
        monkeypatch.setattr(ops_module, name, getattr(me, name))
