"""TEST INFRASTRUCTURE: a PyTorch-CPU stand-in for the C-ABI operators the layer graphs of
``mivos_b200.engine`` use (include/mivos_b200.h), written from the header's contracts.  Monkeypatched
over ``mivos_b200.ops`` by tests/test_s2m_cpu.py and tests/test_engine_cpu.py so that the HOST side of
the engines — weight packing, channel windows of the concat buffers, dilation tables, buffer shapes,
gather orders, the decoder's skip/broadcast plumbing — can be checked against the reference-generated
golden vectors without a GPU.  It says nothing
about the kernels themselves (tests/test_gpu_z_s2m.py does, on an H100) and nothing in the product
package imports it."""
from __future__ import annotations

import torch
import torch.nn.functional as F


def halo_zeros(n, h, w, c, device, dtype=torch.float32):
    return torch.zeros((n, h + 2, w + 2, c), dtype=torch.float32)


def split_k_workspace(device):
    return torch.zeros(16, dtype=torch.uint8)


def _interior(n, h, w):
    m = torch.zeros((n, h + 2, w + 2), dtype=torch.bool)
    m[:, 1:-1, 1:-1] = True
    return m.reshape(-1)


def conv_gemm(x, pc, n, h, w, out, *, in_coff=0, out_coff=0, relu=False, residual=None, res_coff=0, out_relu=None,
              out_relu_coff=0, round_tf32=False, splitk_ws=None):
    rows = n * (h + 2) * (w + 2)
    X = x.reshape(-1, x.shape[-1])[:, in_coff:in_coff + pc.cin_pad].float()
    assert X.shape[0] >= rows and X.shape[1] == pc.cin_pad, (X.shape, rows, pc.cin_pad)
    W = pc.weight.float()  # [taps, cout_pad, cin_pad]
    acc = torch.zeros((rows, pc.cout_pad))
    if pc.taps == 1:
        acc = X[:rows] @ W[0].t()
    else:
        assert pc.taps in (4, 9) and X.shape[0] == rows
        for t in range(pc.taps):
            off = (t // 3 - 1) * (w + 2) + (t % 3 - 1) if pc.taps == 9 else (t - 2) * (w + 2)
            sh = torch.zeros_like(X)
            if off >= 0:
                sh[:rows - off] = X[off:]
            else:
                sh[-off:] = X[:rows + off]
            acc = acc + sh @ W[t].t()
    v = acc[:, :pc.cout] + pc.bias.float()[:pc.cout]
    inner = _interior(n, h, w)
    if residual is not None:
        v = v + residual.reshape(-1, residual.shape[-1])[:rows, res_coff:res_coff + pc.cout]
    if relu:
        v = v.clamp_min(0)
    o = out.reshape(-1, out.shape[-1])
    o[:rows][inner, out_coff:out_coff + pc.cout] = v[inner]
    if out_relu is not None:
        r = out_relu.reshape(-1, out_relu.shape[-1])
        r[:rows][inner, out_relu_coff:out_relu_coff + pc.cout] = v[inner].clamp_min(0)
    return out


def _nchw(halo, n, h, w, c, coff=0):
    return halo[:, 1:-1, 1:-1, coff:coff + c].permute(0, 3, 1, 2).contiguous()


def _windows_to_rows(cols, n, k2, c, ho, wo, out):
    """F.unfold output [n, c*k2, ho*wo] (channel-major, tap-minor) -> matrix rows = HALO rows of the
    (ho, wo) map, columns (tap, channel); halo rows zero."""
    cols = cols.reshape(n, c, k2, ho, wo).permute(0, 3, 4, 2, 1).reshape(n, ho, wo, k2 * c)
    m = out.reshape(n, ho + 2, wo + 2, out.shape[-1])
    m.zero_()
    m[:, 1:-1, 1:-1, :k2 * c] = cols
    return out


def stem_gather_frames(frames, out):
    n, cin, h, w = frames.shape
    return _windows_to_rows(F.unfold(frames, 7, padding=3, stride=2), n, 49, cin, h // 2, w // 2, out)


def gather_s2(x, n, h, w, c, ks, out):
    return _windows_to_rows(F.unfold(_nchw(x, n, h, w, c), ks, padding=ks // 2, stride=2), n, ks * ks, c, h // 2, w // 2, out)


def gather_dilated(x, n, h, w, c, dilation, out):
    return _windows_to_rows(F.unfold(_nchw(x, n, h, w, c), 3, padding=dilation, dilation=dilation), n, 9, c, h, w, out)


def maxpool3x3s2(x, n, h, w, out):
    c = x.shape[-1]
    out[:, 1:-1, 1:-1, :] = F.max_pool2d(_nchw(x, n, h, w, c), 3, 2, 1).permute(0, 2, 3, 1)
    return out


def halo_avgpool_broadcast(x, n, h, w, c, out, *, in_coff=0, out_coff=0):
    m = _nchw(x, n, h, w, c, in_coff).mean(dim=(2, 3))  # [n, c]
    out[:, 1:-1, 1:-1, out_coff:out_coff + c] = m[:, None, None, :]
    return out


def upsample_bilinear(src, n, hs, ws, dst, h, w, c, *, src_coff=0, dst_coff=0):
    up = F.interpolate(_nchw(src, n, hs, ws, c, src_coff), size=(h, w), mode="bilinear", align_corners=False)
    dst[:, 1:-1, 1:-1, dst_coff:dst_coff + c] = up.permute(0, 2, 3, 1)
    return dst


def halo_upsample_to_plane(halo, n, hs, ws, out_h, out_w, *, coff=0, sigmoid=False, out=None):
    up = F.interpolate(_nchw(halo, n, hs, ws, 1, coff), size=(out_h, out_w), mode="bilinear", align_corners=False)
    up = torch.sigmoid(up) if sigmoid else up
    if out is not None:
        out.copy_(up)
        return out
    return up



# ------------------------------------------------------------------ propagation-path operators
def _stem_s2d_frames(frames, out):
    """Header contract of mivos_stem_gather_s2d: out[row(Y,X), py*8*cin + j*cin + c] = in[c, 2Y+py, 2X-4+j]."""
    n, cin, h, w = frames.shape
    ho, wo = h // 2, w // 2
    xp = F.pad(frames, (4, 4, 0, 0))                                   # x index shifted by 4
    m = out.reshape(n, ho + 2, wo + 2, out.shape[-1])
    m.zero_()
    for py in range(2):
        rows = xp[:, :, py::2, :]                                       # [n, cin, ho, w + 8]
        win = rows.unfold(3, 8, 2)[:, :, :, :wo]                        # [n, cin, ho, wo, 8]: x_in = 2X-4+j
        m[:, 1:-1, 1:-1, py * 8 * cin:(py + 1) * 8 * cin] = win.permute(0, 2, 3, 4, 1).reshape(n, ho, wo, 8 * cin)
    return out


def stem_gather(frame, masks, out, s2d=False):
    if s2d:
        if masks is None:
            return _stem_s2d_frames(frame, out)
        if masks.dim() == 5:
            G, k = masks.shape[:2]
            rows = out.shape[0] // (G * k)
            for g in range(G):
                stem_gather(frame[g:g + 1], masks[g], out[g * k * rows:(g + 1) * k * rows], s2d=True)
            return out
        k = masks.shape[0]
        others = masks.sum(0, keepdim=True) - masks
        return _stem_s2d_frames(torch.cat([frame.expand(k, -1, -1, -1), masks, others], 1), out)
    return _stem_gather_im2col(frame, masks, out)


def _stem_gather_im2col(frame, masks, out):
    """masks None: `frame` is a batch [n,3,H,W]; else frame [1,3,H,W] + masks [K,1,H,W] -> K five-channel
    inputs cat(frame, mask_k, sum of the other masks) (prop_net.py:150-157)."""
    if masks is None:
        return stem_gather_frames(frame, out)
    if masks.dim() == 5:  # G groups of (frame, K masks): output images group-major, "others" within a group
        G, k = masks.shape[:2]
        rows = out.shape[0] // (G * k)
        for g in range(G):
            _stem_gather_im2col(frame[g:g + 1], masks[g], out[g * k * rows:(g + 1) * k * rows])
        return out
    k = masks.shape[0]
    others = masks.sum(0, keepdim=True) - masks
    return stem_gather_frames(torch.cat([frame.expand(k, -1, -1, -1), masks, others], 1), out)


def halo_copy(src, dst, n, h, w, c, *, src_coff=0, dst_coff=0, relu=False):
    v = src[:, 1:-1, 1:-1, src_coff:src_coff + c]
    if src.shape[0] != n:  # src_n maps, each broadcast over n / src_n consecutive images
        v = v.repeat_interleave(n // src.shape[0], 0)
    dst[:n, 1:-1, 1:-1, dst_coff:dst_coff + c] = v.clamp_min(0) if relu else v
    return dst


def halo_to_pixels(halo, n, h, w, coff, c, out):
    out.reshape(n, h * w, c).copy_(halo[:n, 1:-1, 1:-1, coff:coff + c].reshape(n, h * w, c))
    return out


def halo_to_nchw(halo, n, h, w, c, coff=0, out=None):
    r = _nchw(halo[:n], n, h, w, c, coff)
    if out is not None:
        out.copy_(r)
        return out
    return r


def nchw_to_halo(x, halo, coff=0, relu=False):
    n, c, h, w = x.shape
    halo[:n, 1:-1, 1:-1, coff:coff + c] = (x.clamp_min(0) if relu else x).permute(0, 2, 3, 1)
    return halo


def bank_from_nchw(keys, values, bank_k, bank_v):
    k, _, t, h, w = keys.shape
    bank_k[:, :t * h * w] = keys.reshape(k, 128, -1).transpose(1, 2)
    bank_v[:, :t * h * w] = values.reshape(k, 512, -1).transpose(1, 2)


def bank_write(halo, k, h, w, coff_k, coff_v, bank_k, bank_v, t, dyn_t=None):
    hw = h * w
    if dyn_t is not None:
        t = int(dyn_t[0])
    bank_k[:, t * hw:(t + 1) * hw] = halo[:k, 1:-1, 1:-1, coff_k:coff_k + 128].reshape(k, hw, 128)
    bank_v[:, t * hw:(t + 1) * hw] = halo[:k, 1:-1, 1:-1, coff_v:coff_v + 512].reshape(k, hw, 512)


def memory_read_workspace_bytes(k, slots, hw, top_k):
    return 16


def memory_read(bank_k, bank_v, slots, qk, top_k, out, *, out_coff=0, halo_hw=None, workspace=None, algo=0,
                want_topk=False, dyn_slots=None, q_div=0):
    """Header contract of mivos_memory_read: per object, affinity of every live slot with every query
    pixel (keys . q / sqrt(128)), top-k over the slots, softmax over the survivors, weighted values.
    Object o reads query set o // q_div of qk [sets,hw,128] (q_div = 0: the one set [hw,128])."""
    k = bank_k.shape[0]
    hw = qk.shape[-2]
    if dyn_slots is not None:  # live slot count read on the device; `slots` is then only the capacity
        slots = int(dyn_slots[0])
    qsets = (qk if qk.dim() == 3 else qk[None]) / (128 ** 0.5)
    res = []
    for o in range(k):
        q = qsets[o // q_div if q_div > 0 else 0]
        aff = bank_k[o, :slots] @ q.t()                      # [slots, hw]
        vals, idx = torch.topk(aff, top_k, dim=0)
        wgt = torch.softmax(vals, dim=0)                     # [k, hw]
        res.append(torch.einsum("kq,kqc->qc", wgt, bank_v[o, :slots][idx]))  # [hw, 512]
    r = torch.stack(res)
    if halo_hw is not None:
        h, w = halo_hw
        out[:k, 1:-1, 1:-1, out_coff:out_coff + 512] = r.reshape(k, h, w, 512)
    else:
        out[:, :, out_coff:out_coff + 512] = r
    return out


def upsample2x_add(x, up, n, h, w, x_relu=None, skip=None):
    u = F.interpolate(_nchw(up, n, h // 2, w // 2, up.shape[-1]), scale_factor=2, mode="bilinear", align_corners=False)
    base = skip[:, 1:-1, 1:-1, :].repeat_interleave(n // skip.shape[0], 0) if skip is not None else x[:n, 1:-1, 1:-1, :]
    v = base + u.permute(0, 2, 3, 1)
    x[:n, 1:-1, 1:-1, :] = v
    if x_relu is not None:
        x_relu[:n, 1:-1, 1:-1, :] = v.clamp_min(0)
    return x


def upsample4x_sigmoid_aggregate(logits, k, h4, w4, coff=0, want_raw=False, want_prob=True, raw_out=None, prob_out=None,
                                 groups=1):
    if groups > 1:  # G independent sets of k objects: aggregation within a set
        hh = logits.shape[1]
        for g in range(groups):
            upsample4x_sigmoid_aggregate(logits[g * k:(g + 1) * k], k, h4, w4, coff, raw_out=None if raw_out is None else raw_out[g * k:(g + 1) * k],
                                         prob_out=None if prob_out is None else prob_out[g])
        return raw_out, prob_out
    lg = F.interpolate(_nchw(logits, k, h4, w4, 1, coff), scale_factor=4, mode="bilinear", align_corners=False)
    raw = torch.sigmoid(lg)
    prob = None
    if want_prob or prob_out is not None:
        bg = torch.prod(1 - raw, dim=0, keepdim=True)
        p = torch.cat([bg, raw], 0).clamp(1e-7, 1 - 1e-7)
        prob = torch.softmax(torch.log(p / (1 - p)), dim=0)
        if prob_out is not None:
            prob_out.copy_(prob)
            prob = prob_out
    if raw_out is not None:
        raw_out.copy_(raw)
        raw = raw_out
    return (raw if (want_raw or raw_out is not None) else None), prob


def fusion_gather(im, seg1, seg2, attn, nc, nr, out_halo):
    h, w = im.shape[-2:]
    t = torch.tensor([nc, nr]).view(1, 2, 1, 1).expand(1, 2, h, w)
    out_halo[:, 1:-1, 1:-1, :9] = torch.cat([im, seg1, seg2, attn, t], 1).permute(0, 2, 3, 1)
    return out_halo



# ------------------------------------------------------------------ runtime operators (InferenceCore)
def store_words(dst64, vals64, dst32=None, vals32=()):
    for i, v in enumerate(vals64):
        dst64[i] = int(v)
    for i, v in enumerate(vals32):
        dst32[i] = int(v)


def copy_segments(fixed, dyn, nbytes, n, dyn_is_src, max_bytes):
    """Header contract of mivos_copy_segments on host memory: the "device pointers" of CPU tensors are addresses."""
    import ctypes
    for i in range(n):
        d, f, b = int(dyn[i]), int(fixed[i]), int(nbytes[i])
        if d == 0:
            continue
        src, dst = (d, f) if dyn_is_src else (f, d)
        ctypes.memmove(dst, src, b)


def store_i32(dst, *vals):
    for i, v in enumerate(vals):
        dst[i] = int(v)


def aggregate_wbg(prob, keep_bg=False, hard=False, const_bg=False):
    bg = torch.full_like(prob[0:1], 0.5) if const_bg else torch.prod(1 - prob, dim=0, keepdim=True)
    p = torch.cat([bg, prob], 0).clamp(1e-7, 1 - 1e-7)
    lg = torch.log(p / (1 - p))
    sm = torch.softmax(lg * 1000 if hard else lg, dim=0)
    return sm if keep_bg else sm[1:]


def argmax_unpad(prob, pad, h, w, masks_padded, masks_out):
    k1, t, _, nh, nw = prob.shape
    m = torch.argmax(prob[:, :, 0], dim=0).to(torch.uint8)  # [t, nh, nw]
    masks_padded.copy_(m.unsqueeze(1))
    if masks_out is not None:
        masks_out.copy_(m[:, pad[2]:pad[2] + h, pad[0]:pad[0] + w])


def attention_map(mk, qk, h16, w16, pos, neg):
    """Header contract of mivos_attention_map: W = softmax over the memory axis of mk . qk / sqrt(128)
    (no top-k), 16x area-pooled pos/neg row vectors @ W, bilinear back to (H, W)."""
    W = torch.softmax(mk @ (qk / (128 ** 0.5)).t(), dim=0)  # [hw_m, hw_q]
    rows = [F.avg_pool2d(m, 16).reshape(1, h16 * w16) @ W for m in (pos, neg)]
    am = torch.cat(rows, 0).reshape(1, 2, h16, w16)
    return F.interpolate(am, size=(16 * h16, 16 * w16), mode="bilinear", align_corners=False)


def attention_weights(mk, qk):
    """Header contract of mivos_attention_weights: W[i, j] = softmax over memory pixels i of mk[i] . qk[j] / sqrt(128)."""
    return torch.softmax(mk @ (qk / (128 ** 0.5)).t(), dim=0)


def halo_sigmoid_to_plane(halo, h, w, coff, plane):
    plane.copy_(torch.sigmoid(halo[0, 1:-1, 1:-1, coff]))
    return plane


OPS = ("halo_zeros", "split_k_workspace", "conv_gemm", "stem_gather_frames", "gather_s2", "gather_dilated", "maxpool3x3s2",
       "halo_avgpool_broadcast", "upsample_bilinear", "halo_upsample_to_plane", "stem_gather", "halo_copy", "halo_to_pixels",
       "halo_to_nchw", "nchw_to_halo", "bank_from_nchw", "bank_write", "memory_read_workspace_bytes", "memory_read",
       "upsample2x_add", "upsample4x_sigmoid_aggregate", "fusion_gather", "store_i32", "store_words", "copy_segments", "aggregate_wbg", "argmax_unpad",
       "attention_map", "attention_weights", "halo_sigmoid_to_plane")


def install(monkeypatch, ops_module):
    import sys
    me = sys.modules[__name__]
    for name in OPS:
        monkeypatch.setattr(ops_module, name, getattr(me, name))


# ------------------------------------------------------------------ a device-free stand-in for torch.cuda
class _FakeStream:
    cuda_stream = 0

    def __init__(self, *a, **k):
        pass

    def wait_stream(self, *a):
        pass

    def wait_event(self, *a):
        pass

    def synchronize(self):
        pass


class _FakeEvent:
    def __init__(self, *a, **k):
        pass

    def record(self, *a):
        pass

    def elapsed_time(self, other):
        return 1.0


def install_host_runtime(monkeypatch):
    """Everything InferenceCore / LockstepSession touch besides the operators: the CUDA-device guard
    (mivos_b200._lib.require_cuda_device), streams, events, pinned memory.  With MIVOS_GRAPH=0 the frame
    loop then runs eagerly on CPU tensors over the emulated operators — the host logic alone."""
    import contextlib

    import mivos_b200
    from mivos_b200 import _lib, ops
    install(monkeypatch, ops)
    monkeypatch.setenv("MIVOS_GRAPH", "0")
    monkeypatch.setattr(_lib, "require_cuda_device", lambda device, who: None)
    monkeypatch.setattr(_lib, "poll_kernel_error", lambda *a: None)
    monkeypatch.setattr(torch.cuda, "Stream", _FakeStream)
    monkeypatch.setattr(torch.cuda, "Event", _FakeEvent)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _FakeStream())
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: self)
    monkeypatch.setattr(torch.Tensor, "record_stream", lambda self, *a, **k: None)
    return mivos_b200
