"""Thin torch-tensor wrappers over the C ABI (include/mivos_b200.h).

PyTorch is used here only for device memory and streams; every op launches hand-written sm_90a
kernels from ``libmivos_b200.so``.  Nothing in this module has a CPU or PyTorch fallback.

Layouts (see the header): HALO = [N, H+2, W+2, C] with a zero border, fp32 (TF32 tensor-core path)
or fp16 (the element type is taken from the tensor's dtype); BANK = slot-major fp32 keys
[K, slots, 128] / values [K, slots, 512].
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib
from ._lib import ConvArgs, check

MEMREAD_AUTO, MEMREAD_EXACT_SIMT, MEMREAD_TCGEN05 = 0, 1, 2


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t: Optional[torch.Tensor]) -> C.c_void_p:
    if t is None:
        return C.c_void_p(0)
    return C.c_void_p(t.data_ptr())


def _req(t: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.MivosError("mivos_b200 ops need CUDA tensors (no CPU fallback)")
    if t.dtype != dtype or not t.is_contiguous():
        raise _lib.MivosError(f"expected contiguous {dtype} tensor, got {t.dtype} contiguous={t.is_contiguous()}")
    return t


def _req_act(t: torch.Tensor) -> torch.Tensor:
    """An activation (HALO map / gathered matrix): contiguous fp32 or fp16."""
    return _req(t, torch.float16 if t.dtype == torch.float16 else torch.float32)


def _f16(t: torch.Tensor) -> int:
    return 1 if t.dtype == torch.float16 else 0


def _same_type(*ts) -> int:
    f = _f16(ts[0])
    for t in ts[1:]:
        if t is not None and _f16(t) != f:
            raise _lib.MivosError("activation maps of one operator must share an element type")
    return f


def store_i32(dst: torch.Tensor, *vals: int) -> None:
    """dst[:len(vals)] = vals (int32 device tensor), stream-ordered, no host buffer to keep alive."""
    _req(dst, torch.int32)
    v = list(vals) + [0] * (4 - len(vals))
    check(_lib.lib().mivos_store_i32(_ptr(dst), len(vals), v[0], v[1], v[2], v[3], _stream()), "mivos_store_i32")


def store_words(dst64: Optional[torch.Tensor], vals64, dst32: Optional[torch.Tensor] = None, vals32=()) -> None:
    """dst64[:len(vals64)] = vals64 (int64 device tensor; any length, 64 words per launch) and dst32[:len(vals32)] =
    vals32 (int32, at most 4), stream-ordered, from launch arguments."""
    vals64, vals32 = list(vals64), list(vals32)
    if dst64 is not None:
        _req(dst64, torch.int64)
    if dst32 is not None:
        _req(dst32, torch.int32)
    v = vals32 + [0] * (4 - len(vals32))
    first = True
    for o in range(0, max(len(vals64), 1), 64):
        chunk = vals64[o:o + 64]
        arr = (C.c_int64 * max(len(chunk), 1))(*chunk)
        n32 = len(vals32) if first else 0
        check(_lib.lib().mivos_store_words(C.c_void_p(dst64.data_ptr() + 8 * o) if chunk else C.c_void_p(0), len(chunk), arr,
                                           _ptr(dst32) if n32 else C.c_void_p(0), n32, v[0], v[1], v[2], v[3], _stream()),
              "mivos_store_words")
        first = False


def copy_segments(fixed: torch.Tensor, dyn: torch.Tensor, nbytes: torch.Tensor, n: int, dyn_is_src: bool, max_bytes: int) -> None:
    """Segment i: nbytes[i] bytes from dyn[i] to fixed[i] (dyn_is_src) or fixed[i] to dyn[i]; the dyn pointers are read
    on the device when the (captured) launch runs.  All three are int64 device tensors."""
    _req(fixed, torch.int64), _req(dyn, torch.int64), _req(nbytes, torch.int64)
    check(_lib.lib().mivos_copy_segments(_ptr(fixed), _ptr(dyn), _ptr(nbytes), n, int(dyn_is_src), int(max_bytes), _stream()),
          "mivos_copy_segments")


def halo_zeros(n: int, h: int, w: int, c: int, device, dtype=torch.float32) -> torch.Tensor:
    """A HALO map; the border stays zero for the lifetime of the buffer."""
    return torch.zeros((n, h + 2, w + 2, c), dtype=dtype, device=device)


def round_tf32(x: torch.Tensor) -> torch.Tensor:
    """Round fp32 to TF32 precision (nearest, ties away — what cvt.rna.tf32.f32 does), so that the
    tensor core's operand truncation is exact."""
    return ((x.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


@dataclass
class PackedConv:
    """Weights of one convolution packed for mivos_conv_gemm: [taps][cout_pad][cin_pad] + bias."""

    weight: torch.Tensor
    bias: torch.Tensor
    cin: int
    cin_pad: int
    cout: int
    cout_pad: int
    taps: int
    ksize: int
    stride: int


def pack_conv(weight: torch.Tensor, bias: Optional[torch.Tensor], bn=None, stride: int = 1,
              im2col: bool = False, device=None, dtype=torch.float32, stem_s2d: bool = False) -> PackedConv:
    """Fold an eval-mode BatchNorm (bn = (gamma, beta, mean, var, eps)) into the convolution and
    pack it K-major for the implicit GEMM.  `im2col=True` flattens (ky, kx, cin) into one K axis
    (used for the 7x7 stem and the stride-2 convs whose input is pre-gathered).  dtype float32:
    weights rounded to TF32, K padded to 32; float16: weights rounded to fp16 (RNE), K padded to 64
    (one 128-byte swizzled k-block either way)."""
    kq = 64 if dtype == torch.float16 else 32
    w = weight.detach().to(torch.float64).cpu()
    cout, cin, kh, kw = w.shape
    b = torch.zeros(cout, dtype=torch.float64) if bias is None else bias.detach().to(torch.float64).cpu()
    if bn is not None:
        gamma, beta, mean, var, eps = bn
        scale = gamma.detach().to(torch.float64).cpu() / torch.sqrt(var.detach().to(torch.float64).cpu() + eps)
        w = w * scale.view(-1, 1, 1, 1)
        b = (b - mean.detach().to(torch.float64).cpu()) * scale + beta.detach().to(torch.float64).cpu()
    cout_pad = (cout + 31) // 32 * 32
    if stem_s2d:
        # 7x7 / stride 2 / pad 3 as four VERTICAL taps dy = -2..1 over the matrix of mivos_stem_gather_s2d:
        # k = py*8*cin + (dx+2)*2*cin + px*cin + c  <->  ky = 2dy+py+3, kx = 2dx+px+3 (weight 0 where an index is -1)
        assert kh == 7 and kw == 7 and stride == 2
        kpad = (16 * cin + kq - 1) // kq * kq
        wp = torch.zeros((4, cout_pad, kpad), dtype=torch.float64)
        for t in range(4):
            for py in range(2):
                ky = 2 * (t - 2) + py + 3
                if ky < 0:
                    continue
                for dxi in range(4):
                    for px in range(2):
                        kx = 2 * (dxi - 2) + px + 3
                        if kx < 0:
                            continue
                        k0 = py * 8 * cin + dxi * 2 * cin + px * cin
                        wp[t, :cout, k0:k0 + cin] = w[:, :, ky, kx]
        taps, cin_pad = 4, kpad
    elif im2col or kh == 1:
        k = kh * kw * cin
        kpad = (k + kq - 1) // kq * kq
        wp = torch.zeros((1, cout_pad, kpad), dtype=torch.float64)
        wp[0, :cout, :k] = w.permute(0, 2, 3, 1).reshape(cout, k)  # (ky, kx, ci) fastest ci
        taps, cin_pad = 1, kpad
    else:
        assert kh == 3 and kw == 3 and stride == 1
        cin_pad = (cin + kq - 1) // kq * kq
        wp = torch.zeros((9, cout_pad, cin_pad), dtype=torch.float64)
        wp[:, :cout, :cin] = w.permute(2, 3, 0, 1).reshape(9, cout, cin)
        taps = 9
    bp = torch.zeros(cout_pad, dtype=torch.float64)
    bp[:cout] = b
    wp = wp.to(torch.float16).contiguous() if dtype == torch.float16 else round_tf32(wp.to(torch.float32).contiguous())
    return PackedConv(wp.to(device), bp.to(torch.float32).to(device),
                      cin, cin_pad, cout, cout_pad, taps, kh, stride)


def conv_gemm(x: torch.Tensor, pc: PackedConv, n: int, h: int, w: int, out: torch.Tensor, *,
              in_coff: int = 0, out_coff: int = 0, relu: bool = False,
              residual: Optional[torch.Tensor] = None, res_coff: int = 0,
              out_relu: Optional[torch.Tensor] = None, out_relu_coff: int = 0,
              round_tf32: bool = False, splitk_ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[HALO (n,h,w)] = conv(x) (+residual)(relu).  `x` is a HALO map of the same (n,h,w) for
    taps=9 / 1x1, or a pre-gathered matrix whose rows are the HALO rows of the output map."""
    _req_act(x), _req_act(out)
    if _f16(x) != _f16(pc.weight):
        raise _lib.MivosError("conv_gemm: input map and packed weights differ in element type")
    rows = n * (h + 2) * (w + 2)
    a = ConvArgs()
    a.in_f16, a.out_f16 = _f16(x), _f16(out)
    a.in_ = x.data_ptr()
    a.in_rows = x.numel() // x.shape[-1]
    a.in_cstride = x.shape[-1]
    a.in_coff = in_coff
    a.n, a.h, a.w = n, h, w
    a.cin_pad = pc.cin_pad
    a.taps = pc.taps
    a.weight = pc.weight.data_ptr()
    a.bias = pc.bias.data_ptr()
    a.cout, a.cout_pad = pc.cout, pc.cout_pad
    a.out = out.data_ptr()
    a.out_cstride = out.shape[-1]
    a.out_coff = out_coff
    assert out.numel() // out.shape[-1] >= rows and a.in_rows >= rows
    _same_type(out, residual, out_relu)
    if residual is not None:
        _req_act(residual)
        a.residual = residual.data_ptr()
        a.res_cstride = residual.shape[-1]
        a.res_coff = res_coff
    if out_relu is not None:
        _req_act(out_relu)
        a.out_relu = out_relu.data_ptr()
        a.out_relu_cstride = out_relu.shape[-1]
        a.out_relu_coff = out_relu_coff
    a.relu = (1 if relu else 0) | (2 if (round_tf32 and not a.out_f16) else 0)
    if splitk_ws is not None:  # zero-initialised scratch (split_k_workspace) owned by this stream's workspace
        a.splitk_ws = splitk_ws.data_ptr()
        a.splitk_ws_bytes = splitk_ws.numel() * splitk_ws.element_size()
    check(_lib.lib().mivos_conv_gemm(C.byref(a), _stream()), "mivos_conv_gemm")
    return out


SPLITK_WS_BYTES = 48 << 20


def split_k_workspace(device) -> torch.Tensor:
    """Scratch for mivos_conv_gemm's split-K path (fp32 partial tiles).  One per stream of launches."""
    return torch.zeros(SPLITK_WS_BYTES, dtype=torch.uint8, device=device)


def stem_gather(frame: torch.Tensor, masks: Optional[torch.Tensor], out: torch.Tensor, s2d: bool = False) -> torch.Tensor:
    """s2d: the space-to-depth matrix of mivos_stem_gather_s2d (16*cin columns, four vertical conv taps) instead
    of the 49-tap im2col matrix.  masks None: `frame` [n,3,H,W] is a batch of frames.  masks [K,1,H,W]: one frame + its K object masks.
    masks [G,K,1,H,W] (any group stride, planes contiguous) with frame [G,3,H,W]: G independent (frame, K
    masks) groups in one launch — the clips of a lock-step step; output images are group-major."""
    _req(frame), _req_act(out)
    h, w = frame.shape[-2:]
    groups, fgs, mgs = 1, 0, 0
    if masks is None:
        k = frame.shape[0]  # a batch of frames
    elif masks.dim() == 5:
        groups, k = masks.shape[0], masks.shape[1]
        if masks.dtype != torch.float32 or not masks[0].is_contiguous() or frame.shape[0] != groups:
            raise _lib.MivosError("stem_gather: grouped masks must be fp32 [G,K,1,H,W] with contiguous groups, frame [G,3,H,W]")
        fgs, mgs = 3 * h * w, masks.stride(0)
    else:
        k = masks.shape[0]
        _req(masks)
    fn = _lib.lib().mivos_stem_gather_s2d if s2d else _lib.lib().mivos_stem_gather
    check(fn(_ptr(frame), _ptr(masks), k, h, w, _ptr(out), out.shape[-1], _f16(out), groups, fgs, mgs, _stream()),
          "mivos_stem_gather_s2d" if s2d else "mivos_stem_gather")
    return out


def gather_s2(x: torch.Tensor, n: int, h: int, w: int, c: int, ks: int, out: torch.Tensor) -> torch.Tensor:
    _req_act(x), _req_act(out)
    check(_lib.lib().mivos_gather_s2(_ptr(x), n, h, w, c, x.shape[-1], ks, _ptr(out), out.shape[-1],
                                     _same_type(x, out), _stream()), "mivos_gather_s2")
    return out


def maxpool3x3s2(x: torch.Tensor, n: int, h: int, w: int, out: torch.Tensor) -> torch.Tensor:
    _req_act(x), _req_act(out)
    assert x.shape[-1] == out.shape[-1]
    check(_lib.lib().mivos_maxpool3x3s2(_ptr(x), n, h, w, x.shape[-1], _ptr(out), _same_type(x, out), _stream()),
          "mivos_maxpool3x3s2")
    return out


def upsample2x_add(x: torch.Tensor, up: torch.Tensor, n: int, h: int, w: int,
                   x_relu: Optional[torch.Tensor] = None, skip: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x += up2x(up); with `skip` (HALO maps [S,...], map j broadcast over images [j*n/S, (j+1)*n/S): a frame's
    skip path over its objects): x = skip + up2x(up)."""
    _req_act(x), _req_act(up)
    assert x.shape[-1] == up.shape[-1]
    skip_n = 1
    if skip is not None:
        _req_act(skip)
        assert skip.shape[-1] == x.shape[-1]
        skip_n = skip.shape[0]
    check(_lib.lib().mivos_upsample2x_add(_ptr(x), _ptr(up), n, h, w, x.shape[-1], _ptr(x_relu), _ptr(skip), skip_n,
                                          _same_type(x, up, x_relu, skip), _stream()), "mivos_upsample2x_add")
    return x


def halo_copy(src: torch.Tensor, dst: torch.Tensor, n: int, h: int, w: int, c: int, *, src_coff: int = 0,
              dst_coff: int = 0, relu: bool = False) -> torch.Tensor:
    _req_act(src), _req_act(dst)
    check(_lib.lib().mivos_halo_copy(_ptr(src), src.shape[0], src.shape[-1], src_coff, _ptr(dst), dst.shape[-1],
                                     dst_coff, n, h, w, c, int(relu), _f16(src), _f16(dst), _stream()),
          "mivos_halo_copy")
    return dst


def halo_to_nchw(halo: torch.Tensor, n: int, h: int, w: int, c: int, coff: int = 0,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req_act(halo)
    if out is None:
        out = torch.empty((n, c, h, w), dtype=torch.float32, device=halo.device)
    check(_lib.lib().mivos_halo_to_nchw(_ptr(halo), n, h, w, halo.shape[-1], coff, c, _ptr(out), _f16(halo),
                                        _stream()), "mivos_halo_to_nchw")
    return out


def nchw_to_halo(x: torch.Tensor, halo: torch.Tensor, coff: int = 0, relu: bool = False) -> torch.Tensor:
    _req(x), _req_act(halo)
    n, c, h, w = x.shape
    check(_lib.lib().mivos_nchw_to_halo(_ptr(x), n, h, w, c, _ptr(halo), halo.shape[-1], coff, int(relu),
                                        _f16(halo), _stream()), "mivos_nchw_to_halo")
    return halo


def halo_to_pixels(halo: torch.Tensor, n: int, h: int, w: int, coff: int, c: int, out: torch.Tensor) -> torch.Tensor:
    _req(halo), _req(out)
    check(_lib.lib().mivos_halo_to_pixels(_ptr(halo), n, h, w, halo.shape[-1], coff, c, _ptr(out), _stream()),
          "mivos_halo_to_pixels")
    return out


def bank_write(halo: torch.Tensor, k: int, h: int, w: int, coff_k: int, coff_v: int,
               bank_k: torch.Tensor, bank_v: torch.Tensor, t: int, dyn_t: Optional[torch.Tensor] = None) -> None:
    """`dyn_t`: optional int32 device scalar holding the bank frame index (CUDA-graph replay); `t`
    is then the largest index that may occur (capacity check only)."""
    _req(halo), _req(bank_k), _req(bank_v)
    check(_lib.lib().mivos_bank_write(_ptr(halo), k, h, w, halo.shape[-1], coff_k, coff_v, _ptr(bank_k),
                                      _ptr(bank_v), bank_k.shape[1], t, _ptr(dyn_t), _stream()), "mivos_bank_write")


def bank_from_nchw(keys: torch.Tensor, values: torch.Tensor, bank_k: torch.Tensor, bank_v: torch.Tensor) -> None:
    """keys [K,128,T,h,w], values [K,512,T,h,w] (reference layout) -> BANK."""
    _req(keys), _req(values), _req(bank_k), _req(bank_v)
    k, _, t, h, w = keys.shape
    check(_lib.lib().mivos_bank_from_nchw(_ptr(keys), _ptr(values), k, t, h * w, _ptr(bank_k), _ptr(bank_v),
                                          bank_k.shape[1], _stream()), "mivos_bank_from_nchw")


def memory_read_workspace_bytes(k: int, slots: int, hw: int, top_k: int) -> int:
    n = _lib.load().mivos_memory_read_workspace(k, slots, hw, top_k)
    if n < 0:
        raise _lib.MivosError(f"memory_read_workspace: bad arguments (k={k} slots={slots} hw={hw} top_k={top_k})")
    return int(n)


def memory_read(bank_k: torch.Tensor, bank_v: torch.Tensor, slots: int, qk: torch.Tensor, top_k: int,
                out: torch.Tensor, *, out_coff: int = 0, halo_hw=None, workspace: Optional[torch.Tensor] = None,
                algo: int = MEMREAD_AUTO, want_topk: bool = False, dyn_slots: Optional[torch.Tensor] = None,
                q_div: int = 0):
    """bank_k [K,cap,128], bank_v [K,cap,512], qk pixel-major [hw,128] — or [sets,hw,128] with q_div objects
    per query set (object o reads set o // q_div: the C clips of a lock-step step in ONE call).  `out` is a
    HALO map (pass halo_hw=(h,w)) or pixel-major [K,hw,C]."""
    _req(bank_k), _req(bank_v), _req(qk), _req_act(out)
    k, cap = bank_k.shape[0], bank_k.shape[1]
    hw = qk.shape[-2]
    if qk.dim() == 3 and (q_div < 1 or (k + q_div - 1) // q_div != qk.shape[0]):
        raise _lib.MivosError(f"memory_read: {qk.shape[0]} query sets for {k} objects need q_div = objects per set (got {q_div})")
    if qk.dim() == 2 and q_div != 0:
        raise _lib.MivosError("memory_read: q_div needs a [sets,hw,128] query tensor")
    need = memory_read_workspace_bytes(k, slots, hw, top_k)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=qk.device)
    idx = val = None
    if want_topk:
        idx = torch.empty((k, hw, top_k), dtype=torch.int32, device=qk.device)
        val = torch.empty((k, hw, top_k), dtype=torch.float32, device=qk.device)
    hh, ww = halo_hw if halo_hw is not None else (0, 0)
    check(_lib.lib().mivos_memory_read(_ptr(bank_k), _ptr(bank_v), cap, k, slots, _ptr(qk), hw, q_div, top_k, _ptr(out),
                                       out.shape[-1], out_coff, hh, ww, _ptr(idx), _ptr(val), _ptr(workspace),
                                       workspace.numel(), algo, _ptr(dyn_slots), _f16(out), _stream()),
          "mivos_memory_read")
    return (out, idx, val) if want_topk else out


def upsample4x_sigmoid_aggregate(logits: torch.Tensor, k: int, h4: int, w4: int, coff: int = 0,
                                 want_raw: bool = False, want_prob: bool = True,
                                 raw_out: Optional[torch.Tensor] = None, prob_out: Optional[torch.Tensor] = None,
                                 groups: int = 1):
    """`groups` G > 1: logits of G*k images (G clips of k objects), prob_out [G,k+1,1,H,W], aggregation per clip."""
    _req(logits)
    dev = logits.device
    lead = (groups,) if groups > 1 else ()
    raw = raw_out if raw_out is not None else (
        torch.empty((groups * k, 1, 4 * h4, 4 * w4), dtype=torch.float32, device=dev) if want_raw else None)
    prob = prob_out if prob_out is not None else (
        torch.empty(lead + (k + 1, 1, 4 * h4, 4 * w4), dtype=torch.float32, device=dev) if want_prob else None)
    if prob is not None:
        _req(prob)
    check(_lib.lib().mivos_upsample4x_sigmoid_aggregate(_ptr(logits), k, h4, w4, logits.shape[-1], coff, _ptr(raw),
                                                        _ptr(prob), groups, _stream()), "mivos_upsample4x_sigmoid_aggregate")
    return raw, prob


def aggregate_wbg(prob: torch.Tensor, keep_bg: bool = False, hard: bool = False, const_bg: bool = False) -> torch.Tensor:
    _req(prob)
    k = prob.shape[0]
    hw = prob[0].numel()
    out = torch.empty((k + 1 if keep_bg else k,) + tuple(prob.shape[1:]), dtype=torch.float32, device=prob.device)
    check(_lib.lib().mivos_aggregate_wbg(_ptr(prob), k, hw, int(keep_bg), int(hard) | (2 if const_bg else 0), _ptr(out), _stream()),
          "mivos_aggregate_wbg")
    return out


def argmax_unpad(prob: torch.Tensor, pad, h: int, w: int, masks_padded: torch.Tensor,
                 masks_out: Optional[torch.Tensor]) -> None:
    """prob [(K+1),T,1,nh,nw] -> masks_padded [T,1,nh,nw] u8 (+ unpadded [T,h,w] u8)."""
    _req(prob), _req(masks_padded, torch.uint8)
    if masks_out is not None:
        _req(masks_out, torch.uint8)
    k1, t, _, nh, nw = prob.shape
    check(_lib.lib().mivos_argmax_unpad(_ptr(prob), k1, t, nh, nw, pad[0], pad[2], h, w, _ptr(masks_padded),
                                        _ptr(masks_out), _stream()), "mivos_argmax_unpad")


def frames_u8_normalize(frames_hwc: torch.Tensor) -> torch.Tensor:
    """u8 [T,H,W,3] on the device -> normalised fp32 [T,3,H,W] (images_to_torch / ToTensor+Normalize)."""
    _req(frames_hwc, torch.uint8)
    t, h, w, c = frames_hwc.shape
    if c != 3:
        raise _lib.MivosError("frames_u8_normalize expects [T,H,W,3]")
    out = torch.empty((t, 3, h, w), dtype=torch.float32, device=frames_hwc.device)
    check(_lib.lib().mivos_frames_u8_normalize(_ptr(frames_hwc), t, h, w, _ptr(out), _stream()), "mivos_frames_u8_normalize")
    return out


def pad2d(x: torch.Tensor, pad) -> torch.Tensor:
    _req(x)
    h, w = x.shape[-2:]
    planes = x.numel() // (h * w)
    out = torch.empty(tuple(x.shape[:-2]) + (h + pad[2] + pad[3], w + pad[0] + pad[1]), dtype=torch.float32,
                      device=x.device)
    check(_lib.lib().mivos_pad2d(_ptr(x), planes, h, w, pad[0], pad[1], pad[2], pad[3], _ptr(out), _stream()),
          "mivos_pad2d")
    return out


def attention_map(mk: torch.Tensor, qk: torch.Tensor, h16: int, w16: int, pos: torch.Tensor,
                  neg: torch.Tensor) -> torch.Tensor:
    """mk, qk pixel-major [hw,128]; pos/neg [1,1,H,W] -> [1,2,H,W]."""
    _req(mk), _req(qk), _req(pos), _req(neg)
    for t in (pos, neg):
        if tuple(t.shape) != (1, 1, 16 * h16, 16 * w16):
            raise _lib.MivosError(f"attention_map: pos/neg {tuple(t.shape)} are not [1,1,{16 * h16},{16 * w16}]")
    out = torch.empty((1, 2, h16 * 16, w16 * 16), dtype=torch.float32, device=mk.device)
    scratch = torch.empty(4 * h16 * w16, dtype=torch.float32, device=mk.device)
    check(_lib.lib().mivos_attention_map(_ptr(mk), _ptr(qk), h16, w16, _ptr(pos), _ptr(neg), _ptr(out),
                                         _ptr(scratch), _stream()), "mivos_attention_map")
    return out


def attention_weights(mk: torch.Tensor, qk: torch.Tensor) -> torch.Tensor:
    """mk, qk pixel-major [hw,128] -> W [hw (memory), hw (query)]: softmax over the memory axis (get_W)."""
    _req(mk), _req(qk)
    hw = mk.shape[0]
    if mk.dim() != 2 or mk.shape[1] != 128 or qk.shape != mk.shape:
        raise _lib.MivosError(f"attention_weights: mk {tuple(mk.shape)} / qk {tuple(qk.shape)} are not both [hw,128]")
    out = torch.empty((hw, hw), dtype=torch.float32, device=mk.device)
    scratch = torch.empty(4 * hw, dtype=torch.float32, device=mk.device)
    check(_lib.lib().mivos_attention_weights(_ptr(mk), _ptr(qk), hw, _ptr(out), _ptr(scratch), _stream()),
          "mivos_attention_weights")
    return out


def fusion_gather(im, seg1, seg2, attn, nc: float, nr: float, out_halo: torch.Tensor) -> torch.Tensor:
    for t in (im, seg1, seg2, attn):
        _req(t)
    _req_act(out_halo)
    h, w = im.shape[-2:]
    check(_lib.lib().mivos_fusion_gather(_ptr(im), _ptr(seg1), _ptr(seg2), _ptr(attn), C.c_float(nc), C.c_float(nr),
                                         h, w, _ptr(out_halo), out_halo.shape[-1], _f16(out_halo), _stream()),
          "mivos_fusion_gather")
    return out_halo


def halo_sigmoid_to_plane(halo: torch.Tensor, h: int, w: int, coff: int, plane: torch.Tensor) -> torch.Tensor:
    _req(halo), _req(plane)
    check(_lib.lib().mivos_halo_sigmoid_to_plane(_ptr(halo), h, w, halo.shape[-1], coff, _ptr(plane), _stream()),
          "mivos_halo_sigmoid_to_plane")
    return plane


# ------------------------------------------------------------------ S2M operators (SURVEY.md 8f-3)
def stem_gather_frames(frames: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """7x7/2 stem windows of a batch of 3- or 6-channel NCHW images -> im2col matrix (rows = HALO rows
    of the half-resolution output map)."""
    _req(frames), _req_act(out)
    n, cin, h, w = frames.shape
    check(_lib.lib().mivos_stem_gather_frames(_ptr(frames), n, cin, h, w, _ptr(out), out.shape[-1], _f16(out), _stream()),
          "mivos_stem_gather_frames")
    return out


def gather_dilated(x: torch.Tensor, n: int, h: int, w: int, c: int, dilation: int, out: torch.Tensor) -> torch.Tensor:
    _req_act(x), _req_act(out)
    check(_lib.lib().mivos_gather_dilated(_ptr(x), n, h, w, c, x.shape[-1], dilation, _ptr(out), out.shape[-1],
                                          _same_type(x, out), _stream()), "mivos_gather_dilated")
    return out


def halo_avgpool_broadcast(x: torch.Tensor, n: int, h: int, w: int, c: int, out: torch.Tensor, *, in_coff: int = 0,
                           out_coff: int = 0) -> torch.Tensor:
    _req_act(x), _req_act(out)
    check(_lib.lib().mivos_halo_avgpool_broadcast(_ptr(x), n, h, w, c, x.shape[-1], in_coff, _ptr(out), out.shape[-1],
                                                  out_coff, _same_type(x, out), _stream()), "mivos_halo_avgpool_broadcast")
    return out


def upsample_bilinear(src: torch.Tensor, n: int, hs: int, ws: int, dst: torch.Tensor, h: int, w: int, c: int, *,
                      src_coff: int = 0, dst_coff: int = 0) -> torch.Tensor:
    _req_act(src), _req_act(dst)
    check(_lib.lib().mivos_upsample_bilinear(_ptr(src), n, hs, ws, src.shape[-1], src_coff, _ptr(dst), h, w, dst.shape[-1],
                                             dst_coff, c, _same_type(src, dst), _stream()), "mivos_upsample_bilinear")
    return dst


def halo_upsample_to_plane(halo: torch.Tensor, n: int, hs: int, ws: int, out_h: int, out_w: int, *, coff: int = 0,
                           sigmoid: bool = False, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One fp32 HALO channel -> [n,1,out_h,out_w] (bilinear, align_corners=False), optional sigmoid."""
    _req(halo)
    if out is None:
        out = torch.empty((n, 1, out_h, out_w), dtype=torch.float32, device=halo.device)
    _req(out)
    check(_lib.lib().mivos_halo_upsample_to_plane(_ptr(halo), n, hs, ws, halo.shape[-1], coff, out_h, out_w, int(sigmoid),
                                                  _ptr(out), _stream()), "mivos_halo_upsample_to_plane")
    return out


# ------------------------------------------------------------------ mask egress (SURVEY.md 8f-4)
# interact/interactive_utils.py:107-117: the GUI's overlay colours for labels 0..6
GUI_OVERLAY_COLORS = ((0, 0, 0), (255, 50, 50), (50, 255, 50), (50, 50, 255), (255, 50, 255), (50, 255, 255), (255, 255, 50))
_overlay_tables = {}


def overlay_davis(image: torch.Tensor, mask: torch.Tensor, alpha: float = 0.5, fade: bool = False,
                  colors=GUI_OVERLAY_COLORS) -> torch.Tensor:
    """image u8 [h,w,3] or [t,h,w,3], mask u8 [h,w] or [t,h,w] (CUDA) -> u8 overlay, same shape as image."""
    _req(image, torch.uint8), _req(mask, torch.uint8)
    if image.shape[-1] != 3 or tuple(image.shape[:-1]) != tuple(mask.shape) or mask.dim() not in (2, 3):
        raise _lib.MivosError(f"overlay_davis: image {tuple(image.shape)} / mask {tuple(mask.shape)} do not match")
    key = (image.device, tuple(map(tuple, colors)))
    tab = _overlay_tables.get(key)
    if tab is None:
        tab = torch.tensor(colors, dtype=torch.uint8).reshape(-1, 3).contiguous().to(image.device)
        _overlay_tables[key] = tab
    t = 1 if mask.dim() == 2 else mask.shape[0]
    h, w = mask.shape[-2:]
    out = torch.empty_like(image)
    check(_lib.lib().mivos_overlay_davis(_ptr(image), _ptr(mask), t, h, w, _ptr(tab), tab.shape[0], float(alpha), int(fade),
                                         _ptr(out), _stream()), "mivos_overlay_davis")
    return out
