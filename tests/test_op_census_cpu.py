"""CPU: the operator census checker (tests/op_census.py) has teeth, and no launch symbol escapes the three censuses.

The emulated operators of tests/abi_emulator*.py pass it on HALO windows of larger allocations, in fp32 and fp16
(forms without an emulator use their float64 reference rounded to fp32).  Each emulated kernel bug fails it: a grouped
aggregation that takes the previous group's last object, "others" of stem_gather_range summed over the chunk only, a
grouped skip broadcast by uniform division, x_relu from the pre-add value, a copy one channel past c, a resize with
align_corners=True, attention softmax over the query axis, a streamed map without one rescale, argmax ties to the
last maximum, an unpad one row off, fusion_gather with nc / nr swapped, an average over the padded pixel count, one
element written into map n at a prefix tick.  The census over an emulated InferenceCore checks every form it called.
Every symbol of mivos_b200._lib.SIGNATURES is claimed by one census or listed in op_census.NOT_CENSUSED."""
import ast
import functools
import os
import re

import pytest
import torch
import torch.nn.functional as F

import abi_emulator as E
import abi_emulator_groups as EG
import abi_emulator_host as EH
import memory_census as MC
import op_census as OC
import op_references as R
from mivos_b200 import _lib, ops

H16, F32 = torch.float16, torch.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _halo(x, cs, coff=0, extra=1, dtype=F32, fill=3.25):
    """x [n, c, h, w] in channels [coff, coff + c) of a HALO map of cs channels: the leading n maps of an allocation
    of n + extra maps filled with a sentinel (the HALO border too)."""
    n, c, h, w = x.shape
    parent = torch.full((n + extra, h + 2, w + 2, cs), fill, dtype=dtype)
    parent[:n, 1:-1, 1:-1, coff:coff + c] = x.permute(0, 2, 3, 1).to(dtype)
    return parent[:n]


def _zero_border(x, cs, coff=0, dtype=F32):
    n, c, h, w = x.shape
    t = torch.zeros((n, h + 2, w + 2, cs), dtype=dtype)
    t[:, 1:-1, 1:-1, coff:coff + c] = x.permute(0, 2, 3, 1).to(dtype)
    return t


def _out(n, h, w, cs, dtype=F32, extra=1):
    return torch.full((n + extra, h + 2, w + 2, cs), -1.5, dtype=dtype)[:n]


def _first(sizes):
    f = [0]
    for k in sizes:
        f.append(f[-1] + k)
    return torch.tensor(f, dtype=torch.int32)


def _logits(maps, h4, w4, seed):
    return R._bilinear(torch.randn(maps, 1, 2, 2, generator=_g(seed)) * 4, h4, w4).float()


# ------------------------------------------------------------------ cases: (form, kernel, args)
def _stem_frames(dtype):
    fr = torch.randn(2, 6, 8, 12, generator=_g(1))
    return "stem_gather_frames", E.stem_gather_frames, (fr, torch.full((2 * 6 * 8 + 9, 320), 9.0, dtype=dtype)[:2 * 6 * 8])


def _others(masks):
    """The kernel's "others": the other masks added to 0 in object order, in fp32."""
    out = []
    for k in range(masks.shape[0]):
        acc = torch.zeros_like(masks[0])
        for j in range(masks.shape[0]):
            if j != k:
                acc = acc + masks[j]
        out.append(acc)
    return torch.stack(out)


def _stem_kernel(frame, masks, out, s2d=False):
    """mivos_stem_gather of one frame and its K masks in the kernel's order of additions."""
    k = masks.shape[0]
    img = torch.cat([frame.expand(k, -1, -1, -1), masks, _others(masks)], 1)
    out.copy_(R.stem_matrix(img.double(), out.shape[-1], s2d).to(out.dtype))
    return out


def _stem_any(frame, masks, out, s2d=False):
    """mivos_stem_gather in all its forms, the mask forms in the kernel's order of additions."""
    if masks is None:
        return E.stem_gather(frame, masks, out, s2d)
    if masks.dim() == 4:
        return _stem_kernel(frame, masks, out, s2d)
    rows = out.shape[0] // (masks.shape[0] * masks.shape[1])
    for g in range(masks.shape[0]):
        k = masks.shape[1]
        _stem_kernel(frame[g:g + 1], masks[g], out[g * k * rows:(g + 1) * k * rows], s2d)
    return out


def _stem_masks(dtype):
    fr = torch.randn(1, 3, 8, 12, generator=_g(2))
    m = torch.rand(4, 1, 8, 12, generator=_g(3))
    return "stem_gather", _stem_kernel, (fr, m, torch.full((4 * 6 * 8 + 5, 96), 9.0, dtype=dtype)[:4 * 6 * 8]), dict(s2d=True)


def _range_kernel(chunk_only=False):
    def stem_gather_range(frame, masks, obj0, n, out):
        src = masks[obj0:obj0 + n] if chunk_only else masks
        others = src.sum(0, keepdim=True) - masks[obj0:obj0 + n]
        img = torch.cat([frame.expand(n, -1, -1, -1), masks[obj0:obj0 + n], others], 1)
        out.copy_(R.stem_matrix(img.double(), out.shape[-1], True).to(out.dtype))
        return out
    return stem_gather_range


def _stem_range(dtype, kernel=None):
    fr = torch.randn(1, 3, 8, 12, generator=_g(4))
    m = torch.rand(20, 1, 8, 12, generator=_g(5))
    return "stem_gather_range", kernel or _range_kernel(), (fr, m, 7, 6, torch.full((6 * 48, 96), 9.0, dtype=dtype))


def _stem_groups(dtype):
    sizes = [2, 1, 3]
    fr = torch.randn(3, 3, 8, 12, generator=_g(6))
    planes = torch.rand(sum(sizes) + 3, 1, 8, 12, generator=_g(7))
    def kernel(frames, planes, n, first, out):
        rows = 6 * 8
        for g, (a, b) in enumerate(zip(first.tolist(), first.tolist()[1:])):
            _stem_kernel(frames[g:g + 1], planes[a + g + 1:b + g + 1], out[a * rows:b * rows], s2d=True)
        return out
    return "stem_gather_groups", kernel, (fr, planes, 6, _first(sizes),
                                                         torch.full((8 * 48, 96), 9.0, dtype=dtype)[:6 * 48])


def _gathers(dtype):
    x = _zero_border(torch.randn(2, 8, 6, 10, generator=_g(8)).relu(), 8, dtype=dtype)
    return [("gather_s2", E.gather_s2, (x, 2, 6, 10, 8, 3, torch.full((2 * 5 * 7 + 3, 72), 9.0, dtype=dtype)[:70])),
            ("gather_dilated", E.gather_dilated, (x, 2, 6, 10, 8, 2, torch.full((2 * 8 * 12 + 3, 72), 9.0, dtype=dtype)[:192])),
            ("maxpool3x3s2", E.maxpool3x3s2, (x, 2, 6, 10, _out(2, 3, 5, 8, dtype)))]


def _fp32_kernel(fn):
    """An emulation whose fp16 maps are computed in fp32 and rounded once on the store, as the kernels do."""
    def kernel(*args, **kw):
        ts = [a for a in list(args) + list(kw.values()) if torch.is_tensor(a) and a.dtype == H16]
        conv = {id(t): t.float() for t in ts}
        r = fn(*[conv.get(id(a), a) for a in args], **{k: conv.get(id(v), v) for k, v in kw.items()})
        for t in ts:
            t.copy_(conv[id(t)])
        return r
    return functools.wraps(fn)(kernel)


def _skip_add(dtype, relu=True):
    x = _halo(torch.randn(4, 8, 6, 10, generator=_g(9)), 8, dtype=dtype)
    up = _zero_border(torch.randn(4, 8, 3, 5, generator=_g(10)), 8, dtype=dtype)
    skip = _zero_border(torch.randn(2, 8, 6, 10, generator=_g(11)), 8, dtype=dtype)
    xr = _out(4, 6, 10, 8, dtype) if relu else None
    return "upsample2x_add", _fp32_kernel(E.upsample2x_add), (x, up, 4, 6, 10), dict(x_relu=xr, skip=skip)


def _skip_add_groups(dtype, kernel=None):
    sizes = [1, 3, 2]
    x = _halo(torch.randn(6, 8, 6, 10, generator=_g(12)), 8, dtype=dtype, extra=2)
    up = _zero_border(torch.randn(6, 8, 3, 5, generator=_g(13)), 8, dtype=dtype)
    skip = _zero_border(torch.randn(3, 8, 6, 10, generator=_g(14)), 8, dtype=dtype)
    return "upsample2x_add_groups", kernel or _fp32_kernel(EG.upsample2x_add_groups), (x, up, 6, 6, 10, skip, _first(sizes)), \
        dict(x_relu=_out(6, 6, 10, 8, dtype))


def _copies(dtype):
    src = _halo(torch.randn(1, 12, 5, 7, generator=_g(15)), 144, 128, dtype=dtype)
    src3 = _halo(torch.randn(3, 12, 5, 7, generator=_g(16)), 140, 128, dtype=dtype)
    x = torch.randn(2, 12, 5, 7, generator=_g(17))
    return [("halo_copy", E.halo_copy, (src, _out(3, 5, 7, 530, dtype), 3, 5, 7, 12), dict(src_coff=128, dst_coff=512)),
            ("halo_copy", E.halo_copy, (src3, _out(3, 5, 7, 24, dtype), 3, 5, 7, 12), dict(src_coff=128, relu=True)),
            ("halo_copy_groups", EG.halo_copy_groups, (src3, _out(4, 5, 7, 530, dtype), 4, 5, 7, 12, _first([1, 2, 1])),
             dict(src_coff=128, dst_coff=512)),
            ("halo_to_nchw", E.halo_to_nchw, (src3, 3, 5, 7, 12), dict(coff=128)),
            ("nchw_to_halo", E.nchw_to_halo, (x, _out(2, 5, 7, 20, dtype)), dict(coff=4, relu=True))]


def _aggregation():
    lg = _halo(_logits(5, 3, 4, 18), 7, 5)
    lg6 = _halo(_logits(6, 3, 4, 19), 7, 5)
    prob = torch.full((3, 6, 1, 12, 16), 2.0)
    p = torch.rand(20, 1, 37, generator=_g(20))
    return [("upsample4x_sigmoid_aggregate", E.upsample4x_sigmoid_aggregate, (lg, 5, 3, 4, 5),
             dict(raw_out=torch.full((6, 1, 12, 16), 2.0)[:5], prob_out=prob[0])),
            ("upsample4x_sigmoid_aggregate_planes", E.upsample4x_sigmoid_aggregate, (lg, 5, 3, 4, 5), dict()),
            ("upsample4x_sigmoid_aggregate_groups", EG.upsample4x_sigmoid_aggregate_groups,
             (lg6, 6, 3, 4, _first([3, 1, 2]), 5), dict(prob_out=torch.full((12, 1, 12, 16), 2.0)[:9])),
            ("aggregate_wbg", E.aggregate_wbg, (p[:4],), dict(keep_bg=True)),
            ("aggregate_wbg", E.aggregate_wbg, (p[:4],), dict(keep_bg=True, hard=True, const_bg=True)),
            ("aggregate_wbg_planes", E.aggregate_wbg, (p,), dict(keep_bg=False))]


def _argmax(kernel=None):
    pr = torch.randint(0, 3, (4, 2, 1, 9, 11), generator=_g(21)).float() / 2
    return "argmax_unpad", kernel or E.argmax_unpad, (pr, (1, 2, 3, 1), 5, 8, torch.full((2, 1, 9, 11), 255, dtype=torch.uint8),
                                                      torch.full((2, 5, 8), 255, dtype=torch.uint8))


def _attn_streamed_map(mk, qk, h16, w16, pos, neg):
    return R.map_reference(mk, qk, h16, w16, pos, neg)[0].float()


def _attn_streamed_weights(mk, qk):
    return torch.cat([W for _a, _b, W, _bd in R.weights_streamed_blocks(mk, qk)], 1).float()


def _attention(scale=1.0):
    g = _g(22)
    mk, qk = torch.randn(63 * 3, 128, generator=g) * scale, torch.randn(63 * 3, 128, generator=g) * scale
    pos, neg = torch.rand(1, 1, 16 * 9, 16 * 21, generator=g), torch.rand(1, 1, 16 * 9, 16 * 21, generator=g)
    return [("attention_map", E.attention_map, (mk, qk, 9, 21, pos, neg)),
            ("attention_weights", E.attention_weights, (mk, qk)),
            ("attention_map_streamed", _attn_streamed_map, (mk, qk, 9, 21, pos, neg)),
            ("attention_weights_streamed", _attn_streamed_weights, (mk, qk))]


def _s2m(dtype, resize=None, pool=None):
    x = _halo(torch.randn(2, 8, 5, 7, generator=_g(23)) * 3, 16, 8, dtype=dtype)
    pl = _halo(torch.randn(2, 1, 5, 7, generator=_g(24)) * 3, 7, 5)
    planes = torch.full((4, 1, 20, 28), 2.0)
    return [("upsample_bilinear", resize or E.upsample_bilinear, (x, 2, 5, 7, _out(2, 13, 11, 24, dtype), 13, 11, 8),
             dict(src_coff=8, dst_coff=16)),
            ("halo_avgpool_broadcast", pool or E.halo_avgpool_broadcast, (x, 2, 5, 7, 8, _out(2, 5, 7, 24, dtype)),
             dict(in_coff=8, out_coff=8)),
            ("halo_upsample_to_plane", E.halo_upsample_to_plane, (pl, 2, 5, 7, 20, 28), dict(coff=5, sigmoid=True,
                                                                                          out=planes[1:3])),
            ("halo_upsample_to_plane", E.halo_upsample_to_plane, (pl, 2, 5, 7, 20, 28), dict(coff=5))]


def _fusion_kernel(im, seg1, seg2, attn, nc, nr, out_halo):
    """mivos_fusion_gather: nine planes, zeros in the channels past them."""
    h, w = im.shape[-2:]
    out_halo[:1, 1:h + 1, 1:w + 1, 9:] = 0
    return E.fusion_gather(im, seg1, seg2, attn, nc, nr, out_halo)


def _normalize(frames_hwc):
    x = frames_hwc.permute(0, 3, 1, 2).float() / 255
    return (x - torch.tensor(OC.NORM_MEAN).view(1, 3, 1, 1)) / torch.tensor(OC.NORM_STD).view(1, 3, 1, 1)


def _pad2d(x, pad):
    return F.pad(x, pad)


def _misc(dtype, fusion=None):
    g = _g(25)
    im, s1, s2, at = (torch.rand(1, c, 7, 9, generator=g) for c in (3, 1, 1, 2))
    lg = _halo(torch.randn(1, 1, 7, 9, generator=g) * 9, 6, 5)
    u8 = torch.randint(0, 256, (2, 5, 7, 3), generator=g, dtype=torch.uint8)
    return [("fusion_gather", fusion or _fusion_kernel, (im, s1, s2, at, 0.3, 0.7, _out(1, 7, 9, 16, dtype))),
            ("halo_sigmoid_to_plane", E.halo_sigmoid_to_plane, (lg, 7, 9, 5, torch.full((64,), 2.0)[:63].view(7, 9))),
            ("halo_to_pixels", E.halo_to_pixels, (lg, 1, 7, 9, 5, 1, torch.full((70,), 2.0)[:63].view(63, 1))),
            ("frames_u8_normalize", _normalize, (u8,)),
            ("pad2d", _pad2d, (torch.randn(2, 3, 5, 7, generator=g), (1, 2, 3, 4))),
            ("store_words", E.store_words, (torch.full((9,), -7, dtype=torch.int64), [3, -4, 1 << 40]),
             dict(dst32=torch.full((5,), -7, dtype=torch.int32), vals32=(1, 2))),
            ("bank_from_nchw", E.bank_from_nchw, (torch.randn(2, 128, 2, 3, 4, generator=g),
                                                  torch.randn(2, 512, 2, 3, 4, generator=g),
                                                  torch.full((2, 30, 128), 2.0), torch.full((2, 30, 512), 2.0)))]


def _segments(direction_src: bool, kernel=None):
    """copy_segments on host memory (the emulator's "device addresses" are addresses): three 48-byte segments, the
    middle one null, between two buffers inside larger allocations."""
    fixed_buf = torch.full((256,), 7, dtype=torch.uint8)
    dyn_buf = torch.arange(256, dtype=torch.int64).to(torch.uint8)
    fx = [fixed_buf.data_ptr() + 32 + 64 * i for i in range(3)]
    dy = [dyn_buf.data_ptr() + 16 + 64 * i for i in range(3)]
    dy[1] = 0
    t = lambda v: torch.tensor(v, dtype=torch.int64)  # noqa: E731
    return "copy_segments", kernel or E.copy_segments, (t(fx), t(dy), t([48, 48, 48]), 3, direction_src, 48), {}, \
        (fixed_buf, dyn_buf)


def _host_block(k1, T, nh, nw, h, w):
    """A host volume laid out as HostResults: prob [(K+1), T, nh, nw] fp32, padded and unpadded labels, registered."""
    plane = nh * nw
    sizes = (k1 * T * plane * 4, T * plane, T * h * w)
    block = torch.full((sum(sizes),), 0xA5, dtype=torch.uint8)
    return block, (0, sizes[0], sizes[0] + sizes[1])


def _delivery(kernel=None, ti=1):
    """Two clips of K = 2 at frame ti: clip 0 to a host volume, clip 1 a null record."""
    k1, T, nh, nw, h, w, pad = 3, 3, 8, 12, 5, 9, (2, 1, 1, 2)
    block, (op, ol, ou) = _host_block(k1, T, nh, nw, h, w)
    base = EH.host_register(block)
    plane = nh * nw
    rec = [base + op + ti * plane * 4, T * plane, base + ol + ti * plane, base + ou + ti * h * w, 0 | (k1 << 32),
           pad[0] | (pad[2] << 32), h | (w << 32), 0]
    table = torch.tensor(rec + [0] * 8, dtype=torch.int64)
    planes = torch.rand(2 * k1, 1, nh, nw, generator=_g(30))
    planes[:3, 0, 0, :4] = 2.0  # ties: the first maximum wins
    return "deliver_planes", kernel or EH.deliver_planes, (planes, table, 2, nh, nw), {}, [(base, block)]


def _overlay(image, mask, alpha=0.5, fade=False, colors=ops.GUI_OVERLAY_COLORS):
    """mivos_overlay_davis in the kernel's double operations."""
    img, m = image.double(), mask.long()
    tab = torch.tensor(colors, dtype=torch.uint8).reshape(-1, 3).double()
    blend = (img * alpha + (1.0 - alpha) * tab[torch.where(m < tab.shape[0], m, 0)]).trunc()
    obj = m > 0
    nb = torch.zeros_like(obj)
    nb[1:] |= obj[:-1]
    nb[:-1] |= obj[1:]
    nb[:, 1:] |= obj[:, :-1]
    nb[:, :-1] |= obj[:, 1:]
    rest = (img * 0.6).trunc() if fade else img
    return torch.where(obj[..., None], blend, torch.where(nb[..., None], 0.0, rest)).to(torch.uint8)


def _overlay_case(fade):
    g = _g(31)
    image = torch.randint(0, 256, (9, 11, 3), generator=g, dtype=torch.uint8)
    mask = torch.randint(0, 9, (9, 11), generator=g, dtype=torch.uint8) * (torch.rand(9, 11, generator=g) < 0.4)
    return "overlay_davis", _overlay, (image, mask.to(torch.uint8)), dict(alpha=0.3, fade=fade)


def _all(dtype):
    cases = [_stem_frames(dtype), _stem_masks(dtype), _stem_range(dtype), _stem_groups(dtype), _skip_add(dtype),
             _skip_add_groups(dtype)] + _gathers(dtype) + _copies(dtype) + _s2m(dtype) + _misc(dtype)
    if dtype == F32:
        cases += _aggregation() + [_argmax()] + _attention() + [_segments(True), _segments(False), _delivery(),
                                                                 _overlay_case(False), _overlay_case(True)] + [
            ("stem_gather_frames_tiled", E.stem_gather_frames, _stem_frames(dtype)[2])]
    return cases


def _run(case):
    name, fn, args, *kw = case
    hosts = kw[1] if name == "deliver_planes" else ()
    return OC.checked(name, fn, args, kw[0] if kw else {}, hosts=hosts)[1]


# ------------------------------------------------------------------ the emulators pass
@pytest.mark.parametrize("dtype", [F32, H16], ids=["f32", "f16"])
def test_emulated_operators_pass(dtype):
    recs = [_run(c) for c in _all(dtype)]
    assert all(r["ratio"] <= 1.0 for r in recs)
    if dtype == F32:
        assert {r["form"] for r in recs} == set(OC.FORMS)
        groups = [r for r in recs if r["form"] == "upsample4x_sigmoid_aggregate_groups"][0]
        assert groups["group_sizes"] == (3, 1, 2) and groups["prefix"]


# ------------------------------------------------------------------ mutations fail
def _fails(case, match=None):
    with pytest.raises(AssertionError, match=match):
        _run(case)


def test_grouped_aggregation_with_the_previous_groups_last_object_fails():
    def kernel(logits, n, h4, w4, first, coff=0, raw_out=None, prob_out=None):
        f = [int(v) for v in first]
        shifted = torch.tensor([f[0]] + [max(f[0], v - 1) if 0 < i < len(f) - 1 else v for i, v in enumerate(f)][1:],
                               dtype=torch.int32)
        EG.upsample4x_sigmoid_aggregate_groups(logits, n, h4, w4, first, coff, raw_out=raw_out, prob_out=prob_out)
        tmp = torch.empty_like(prob_out)
        EG.upsample4x_sigmoid_aggregate_groups(logits, n, h4, w4, shifted, coff, prob_out=tmp)
        hw = 16 * h4 * w4
        for g, (a, b) in enumerate(zip(f, f[1:])):  # each group's planes from the shifted aggregation's objects
            if g:
                prob_out.reshape(-1)[(a + g + 1) * hw:(b + g + 1) * hw] = tmp.reshape(-1)[(a + g) * hw:(b + g) * hw]
        return raw_out, prob_out
    name, _k, args, kw = _aggregation()[2]
    _fails((name, kernel, args, kw))


def test_stem_gather_range_others_over_the_chunk_fails():
    _fails(_stem_range(F32, _range_kernel(chunk_only=True)), "stem_gather_range: .* exceeds the bound")


def test_grouped_skip_by_uniform_division_fails():
    def kernel(x, up, n, h, w, skip, first, x_relu=None):
        return E.upsample2x_add(x, up, n, h, w, x_relu=x_relu, skip=skip[torch.arange(n) * skip.shape[0] // n])
    _fails(_skip_add_groups(F32, kernel))


def test_x_relu_from_the_pre_add_value_fails():
    def kernel(x, up, n, h, w, x_relu=None, skip=None):
        pre = skip.repeat_interleave(n // skip.shape[0], 0)
        E.upsample2x_add(x, up, n, h, w, skip=skip)
        x_relu[:n, 1:-1, 1:-1] = pre[:, 1:-1, 1:-1].clamp_min(0)
        return x
    name, _k, args, kw = _skip_add(F32)
    _fails((name, kernel, args, kw), "x_relu")


def test_halo_copy_one_channel_past_c_fails():
    def kernel(src, dst, n, h, w, c, *, src_coff=0, dst_coff=0, relu=False):
        return E.halo_copy(src, dst, n, h, w, c + 1, src_coff=src_coff, dst_coff=dst_coff, relu=relu)
    name, _k, args, kw = _copies(F32)[0]
    _fails((name, kernel, args, kw), "outside its window")


def test_resize_with_align_corners_fails():
    def kernel(src, n, hs, ws, dst, h, w, c, *, src_coff=0, dst_coff=0):
        v = src[:n, 1:hs + 1, 1:ws + 1, src_coff:src_coff + c].permute(0, 3, 1, 2)
        up = F.interpolate(v, size=(h, w), mode="bilinear", align_corners=True)
        dst[:n, 1:h + 1, 1:w + 1, dst_coff:dst_coff + c] = up.permute(0, 2, 3, 1)
        return dst
    _fails(_s2m(F32, resize=kernel)[0], "exceeds the bound")


def test_attention_over_the_query_axis_fails():
    def kernel(mk, qk):
        return torch.softmax(mk @ (qk / 128 ** 0.5).t(), dim=1)
    name, _k, args = _attention(4.0)[1]
    _fails((name, kernel, args), "exceeds the bound")


def _map_skipping_one_rescale(mk, qk, h16, w16, pos, neg, skip=1):
    """attention_map_streamed in float64 over key tiles of 128 with an online softmax, where the running sums are not
    rescaled when tile `skip` raises the maximum (every other tile rescales)."""
    hw = mk.shape[0]
    L = mk.double() @ qk.double().t() / 128 ** 0.5
    pooled = torch.cat([F.avg_pool2d(pos.double(), 16), F.avg_pool2d(neg.double(), 16)], 1).reshape(2, hw)
    m = torch.full((hw,), -float("inf"), dtype=torch.float64)
    s, p = torch.zeros(hw, dtype=torch.float64), torch.zeros(2, hw, dtype=torch.float64)
    for t, k0 in enumerate(range(0, hw, R.SK)):
        Lt = L[k0:k0 + R.SK]
        mn = torch.maximum(m, Lt.max(0).values)
        c = torch.ones_like(m) if t == skip else torch.exp(m - mn)
        e = torch.exp(Lt - mn)
        s, p, m = s * c + e.sum(0), p * c + pooled[:, k0:k0 + R.SK] @ e, mn
    mp = (p / s).reshape(1, 2, h16, w16)
    return F.interpolate(mp, size=(16 * h16, 16 * w16), mode="bilinear", align_corners=False).float()


def test_streamed_map_skipping_one_tiles_rescale_fails():
    name, _k, args = _attention(4.0)[2]
    assert _map_skipping_one_rescale(*args, skip=-1).double().sub(
        R.map_reference(*args)[0]).abs().max() < 1e-5  # with every rescale it is the streamed map
    _fails((name, _map_skipping_one_rescale, args), "exceeds the bound")


def test_argmax_ties_to_the_last_maximum_fails():
    def kernel(prob, pad, h, w, masks_padded, masks_out):
        flipped = torch.argmax(prob.flip(0), 0)
        E.argmax_unpad(prob, pad, h, w, masks_padded, masks_out)
        masks_padded.copy_((prob.shape[0] - 1 - flipped).to(torch.uint8))
    _fails(_argmax(kernel), "masks_padded")


def test_unpad_one_row_off_fails():
    def kernel(prob, pad, h, w, masks_padded, masks_out):
        E.argmax_unpad(prob, (pad[0], pad[1], pad[2] + 1, pad[3] - 1), h, w, masks_padded, masks_out)
    _fails(_argmax(kernel), "masks_out")


def test_fusion_gather_with_nc_nr_swapped_fails():
    def kernel(im, seg1, seg2, attn, nc, nr, out_halo):
        return _fusion_kernel(im, seg1, seg2, attn, nr, nc, out_halo)
    _fails(_misc(F32, fusion=kernel)[0], "fusion_gather")


def test_average_over_the_padded_pixel_count_fails():
    def kernel(x, n, h, w, c, out, *, in_coff=0, out_coff=0):
        m = x[:n, :, :, in_coff:in_coff + c].sum((1, 2)) / ((h + 2) * (w + 2))
        out[:n, 1:-1, 1:-1, out_coff:out_coff + c] = m[:, None, None, :].to(out.dtype)
        return out
    _fails(_s2m(F32, pool=kernel)[1], "exceeds the bound")


def test_one_element_into_map_n_at_a_prefix_tick_fails():
    def kernel(x, up, n, h, w, skip, first, x_relu=None):
        EG.upsample2x_add_groups(x, up, n, h, w, skip, first, x_relu=x_relu)
        x.as_strided((1,), (1,), x.storage_offset() + x.numel() + 100).fill_(0.5)  # map n of the allocation
        return x
    _fails(_skip_add_groups(F32, kernel), "outside its window")


def test_copy_segments_dropping_the_last_16_bytes_fails():
    def kernel(fixed, dyn, nbytes, n, dyn_is_src, max_bytes):
        return E.copy_segments(fixed, dyn, nbytes - 16, n, dyn_is_src, max_bytes)
    for direction in (True, False):
        _fails(_segments(direction, kernel), "copy_segments segment")


def test_copy_segments_writing_a_null_segment_fails():
    def kernel(fixed, dyn, nbytes, n, dyn_is_src, max_bytes):
        E.copy_segments(fixed, dyn, nbytes, n, dyn_is_src, max_bytes)
        import ctypes
        ctypes.memset(int(fixed[1]), 0, 16)  # the null segment's fixed destination
    _fails(_segments(True, kernel), "null")


def test_deliver_planes_to_frame_ti_plus_1_fails():
    def kernel(planes, table, clips, nh, nw):
        t = table.clone()
        t[0] += nh * nw * 4
        t[2] += nh * nw
        return EH.deliver_planes(planes, t, clips, nh, nw)
    _fails(_delivery(kernel), "outside its window")


def test_deliver_planes_ties_to_the_last_maximum_fails():
    def kernel(planes, table, clips, nh, nw):
        EH.deliver_planes(planes, table, clips, nh, nw)
        flat = planes.reshape(-1, nh * nw)[:3]
        lab = (2 - torch.argmax(flat.flip(0), 0)).to(torch.uint8)
        EH._at(int(table[2]), nh * nw, torch.uint8).copy_(lab)
    _fails(_delivery(kernel), "padded labels")


def test_overlay_without_the_contour_fails():
    def kernel(image, mask, alpha=0.5, fade=False, colors=ops.GUI_OVERLAY_COLORS):
        out = _overlay(image, mask, alpha, fade, colors)
        keep = (mask == 0)[..., None]
        return torch.where(keep & (out == 0), (image.double() * 0.6).trunc().to(torch.uint8) if fade else image, out)
    name, _k, args, kw = _overlay_case(True)
    _fails((name, kernel, args, kw), "overlay_davis")


# ------------------------------------------------------------------ a real session
def test_census_records_an_emulated_session(monkeypatch, prop_sd, fuse_sd):
    """InferenceCore at 64x96 with K = 3 on the emulated operators, two interactions (the second fuses), through
    OpCensus.record: every operator form the session called is checked, and the wrappers are removed afterwards."""
    mv = E.install_host_runtime(monkeypatch)
    from oracle import weights as Wt
    net = mv.PropagationNetwork(top_k=20, act_dtype=F32)
    net.load_state_dict(prop_sd, strict=True)
    fuse = mv.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    clip, m0 = Wt.synthetic_clip(4, 64, 96, 3, seed=64)
    called, counting = set(), {}

    def count(name, fn):
        @functools.wraps(fn)
        def launch(*a, **k):
            called.add(name)
            return fn(*a, **k)
        return launch
    for name in OC.FORMS:
        counting[name] = count(name, getattr(ops, name))
        monkeypatch.setattr(ops, name, counting[name])
    monkeypatch.setattr(ops, "stem_gather", count("stem_gather", _stem_any))
    counting["stem_gather"] = ops.stem_gather
    census = OC.OpCensus()
    core = mv.InferenceCore(net, fuse, clip, 3, mem_freq=2, device="cpu")
    with census.record("core64"):
        core.interact(m0, 0)
        core.interact(m0.flip(-1).contiguous(), 2)
    assert called and census.checked["core64"] > 0
    assert {r["form"] for r in census.records} == called
    assert all(r["ratio"] <= 1.0 for r in census.records)
    assert all(getattr(ops, n) is counting[n] for n in OC.FORMS)
    print("\n" + census.table() + "\n" + census.summary())


# ------------------------------------------------------------------ nothing escapes
def _ops_symbols() -> dict:
    """ops function -> the mivos_* symbols its body names."""
    src = open(os.path.join(ROOT, "mivos_b200", "ops.py")).read()
    return {node.name: set(re.findall(r"mivos_[a-z0-9_]+", ast.get_source_segment(src, node)))
            for node in ast.parse(src).body if isinstance(node, ast.FunctionDef)}


def _package_uses() -> set:
    """Names used as ops.<name> anywhere in mivos_b200/, interact/ and model/."""
    used = set()
    for d in ("mivos_b200", "interact", "model"):
        for base, _dirs, files in os.walk(os.path.join(ROOT, d)):
            for f in files:
                if f.endswith(".py"):
                    for node in ast.walk(ast.parse(open(os.path.join(base, f)).read())):
                        if isinstance(node, ast.Attribute) and isinstance(node.value, ast.Name) and node.value.id == "ops":
                            used.add(node.attr)
    return used


def _definition(src: str, sym: str):
    """The body of the extern "C" definition of sym in src (braces matched), or None."""
    m = re.search(rf"MIVOS_API [\w ]+\*? ?{sym}\([^;{{]*\{{", src)
    if m is None:
        return None
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(src[i], 0)
        i += 1
    return src[m.end():i - 1]


def test_every_launch_symbol_is_censused_or_listed():
    syms = _ops_symbols()
    claims = {}
    for census, forms in (("conv", OC.CONV_FORMS), ("memory", tuple(MC.READS) + tuple(MC.WRITES)),
                          ("operator", tuple(OC.FORMS))):
        for name in forms:
            for s in syms[name] & set(_lib.SIGNATURES):
                if s in ("mivos_stem_frames_plan", "mivos_attention_plan"):
                    continue
                claims.setdefault(s, []).append(census)
    twice = {s: c for s, c in claims.items() if len(c) > 1}
    assert not twice, f"claimed by more than one census: {twice}"
    unclaimed = set(_lib.SIGNATURES) - set(claims) - set(OC.NOT_CENSUSED)
    assert not unclaimed, f"launch symbols no census checks and NOT_CENSUSED does not list: {sorted(unclaimed)}"
    stale = set(OC.NOT_CENSUSED) & set(claims)
    assert not stale, f"listed in NOT_CENSUSED but censused: {sorted(stale)}"
    assert set(OC.NOT_CENSUSED) <= set(_lib.SIGNATURES)
    used = _package_uses()
    csrc = "".join(open(os.path.join(ROOT, "mivos_b200", "csrc", f)).read()
                   for f in sorted(os.listdir(os.path.join(ROOT, "mivos_b200", "csrc"))) if f.endswith(".cu"))
    for s, why in OC.NOT_CENSUSED.items():
        assert why.startswith(OC.NOT_CENSUSED_REASONS), f"{s}: {why!r} is not a reason to leave a symbol uncensused"
        if why.startswith("no kernel launch"):  # its definition launches nothing
            body = _definition(csrc, s)
            assert body is not None, f"{s}: definition not found"
            assert not re.search(r"launch_pdl|<<<|cudaLaunch|MIVOS_LAUNCHED", body), f"{s} launches a kernel"
        callers = {f for f, ss in syms.items() if s in ss}
        if why.startswith("not launched by the package"):
            assert not callers & used, f"{s} is listed as not launched, but the package calls {callers & used}"
    for name in OC.FORMS:  # every census form is a leaf: it calls a launch symbol itself
        assert syms[name] & set(_lib.SIGNATURES), name
