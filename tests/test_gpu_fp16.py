"""GPU: the fp16 element type of the HALO operators (include/mivos_b200.h: `in_f16` / `out_f16` /
`f16` flags).  fp16 is the precision the reference GUI runs the network in (autocast,
interactive_gui.py:990).  Convolutions are compared against an fp64 convolution of the SAME
fp16-rounded operands: the kernel must be exact up to fp32 accumulation order (2e-5 of the output
range) plus, for fp16 outputs, one round-to-nearest-even of the result (2^-11 relative).  Copies,
max pooling and type conversions are bit-exact."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402

H16 = torch.float16


def _border_kept(out):
    """HALO invariant: no kernel writes the one-pixel border of a map (the 7 sentinel survives), so a border the owner
    zeroed stays zero.  Both the epilogue and the split-K second pass store interior rows only."""
    for b in (out[:, 0], out[:, -1], out[:, :, 0], out[:, :, -1]):
        if not bool((b == 7).all()):
            return False
    return True


def to_halo(x, cpad=None, dtype=H16):
    n, c, h, w = x.shape
    hb = torch.zeros((n, h + 2, w + 2, cpad or c), device=x.device, dtype=dtype)
    hb[:, 1:-1, 1:-1, :c] = x.permute(0, 2, 3, 1).to(dtype)
    return hb


def from_halo(hb, c):
    return hb[:, 1:-1, 1:-1, :c].permute(0, 3, 1, 2).contiguous()


@pytest.mark.parametrize("n,h,w,cin,cout,ks,relu,res,dual,out32", [
    (1, 30, 54, 64, 64, 3, False, False, False, False),
    (1, 30, 54, 256, 1, 3, False, False, False, True),      # decoder.pred: fp16 in, fp32 logits out
    (1, 30, 54, 256, 64, 1, True, False, False, False),
    (2, 60, 108, 128, 128, 3, True, True, False, False),
    (1, 120, 216, 256, 256, 3, False, False, True, False),  # BN=256, dual output
    (1, 30, 54, 1024, 640, 1, False, False, False, True),   # key|value projection: fp32 out
    (1, 7, 5, 64, 32, 3, False, False, False, False),
    (1, 120, 216, 64, 128, 1, True, True, True, False),
    (1, 240, 432, 64, 20, 3, False, False, False, False),   # ragged channel tail
    (8, 30, 54, 1024, 256, 1, True, False, False, False),   # batched 1/16 layer
])
def test_conv_gemm_fp16(dev, n, h, w, cin, cout, ks, relu, res, dual, out32):
    g = torch.Generator(device="cpu").manual_seed(cin * 11 + cout)
    x = torch.randn((n, cin, h, w), generator=g).to(dev)
    wt = (torch.randn((cout, cin, ks, ks), generator=g) / (cin * ks * ks) ** 0.5).to(dev)
    b = torch.randn((cout,), generator=g).to(dev)
    pc = ops.pack_conv(wt, b, device=dev, dtype=H16)
    assert pc.weight.dtype == H16 and pc.cin_pad % 64 == 0
    xin = to_halo(x, pc.cin_pad)
    odt = torch.float32 if out32 else H16
    out = torch.full((n, h + 2, w + 2, pc.cout_pad), 7.0, device=dev, dtype=odt)
    r = torch.randn((n, cout, h, w), generator=g).to(dev) if res else None
    out2 = torch.zeros_like(out) if dual else None
    ops.conv_gemm(xin, pc, n, h, w, out, relu=relu, residual=to_halo(r, pc.cout_pad, odt) if res else None, out_relu=out2)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    got = from_halo(out, cout).double()
    y = F.conv2d(x.half().double(), wt.half().double(), b.double(), padding=ks // 2)
    if res:
        y = y + r.to(odt).double()
    y = y.relu() if relu else y
    scale = float(y.abs().max())
    tol = 2e-5 * scale if out32 else 2e-5 * scale + 2.0 ** -11 * y.abs()
    assert bool(((got - y).abs() <= tol).all())
    assert _border_kept(out)
    if pc.cout_pad > cout:
        assert bool((out[:, 1:-1, 1:-1, cout:] == 7).all())
    if dual:
        assert torch.equal(from_halo(out2, cout), from_halo(out, cout).relu())


def test_mixed_type_rejected(dev):
    wt = torch.randn(64, 64, 3, 3, device=dev)
    pc = ops.pack_conv(wt, None, device=dev, dtype=H16)
    x32 = torch.zeros((1, 10, 10, 64), device=dev)
    out = torch.zeros((1, 10, 10, 64), device=dev, dtype=H16)
    with pytest.raises(_lib.MivosError):
        ops.conv_gemm(x32, pc, 1, 8, 8, out)
    with pytest.raises(_lib.MivosError):  # residual must have the output's element type
        ops.conv_gemm(x32.half(), pc, 1, 8, 8, out, residual=torch.zeros((1, 10, 10, 64), device=dev))


def test_gathers_and_pool_fp16(dev):
    n, c, h, w = 2, 64, 60, 108
    x = torch.randn(n, c, h, w, device=dev).relu().half()
    xh = to_halo(x)
    out = torch.zeros((n, h // 2 + 2, w // 2 + 2, c), device=dev, dtype=H16)
    ops.maxpool3x3s2(xh, n, h, w, out)
    assert torch.equal(from_halo(out, c), F.max_pool2d(x.float(), 3, 2, 1).half())
    for ks, cout in ((3, 96), (1, 128)):
        wt = torch.randn(cout, c, ks, ks, device=dev) / (c * ks * ks) ** 0.5
        b = torch.randn(cout, device=dev)
        pc = ops.pack_conv(wt, b, stride=2, im2col=True, device=dev, dtype=H16)
        gm = torch.zeros((n * (h // 2 + 2) * (w // 2 + 2), pc.cin_pad), device=dev, dtype=H16)
        ops.gather_s2(xh, n, h, w, c, ks, gm)
        o = torch.zeros((n, h // 2 + 2, w // 2 + 2, pc.cout_pad), device=dev)  # fp32 out: isolates the gather
        ops.conv_gemm(gm, pc, n, h // 2, w // 2, o)
        ref = F.conv2d(x.double(), wt.half().double(), b.double(), stride=2, padding=ks // 2)
        assert float((from_halo(o, cout).double() - ref).abs().max()) <= 2e-5 * float(ref.abs().max())
    H, W, K = 96, 160, 3
    fr = torch.randn(1, 3, H, W, device=dev)
    mk = torch.rand(K, 1, H, W, device=dev)
    ws = torch.randn(64, 5, 7, 7, device=dev) / 15
    for masks, wsel, kk in ((mk, ws, K), (None, ws[:, :3].contiguous(), 1)):
        pcs = ops.pack_conv(wsel, None, stride=2, im2col=True, device=dev, dtype=H16)
        gs = torch.zeros((kk * (H // 2 + 2) * (W // 2 + 2), pcs.cin_pad), device=dev, dtype=H16)
        ops.stem_gather(fr, masks, gs)
        o = torch.zeros((kk, H // 2 + 2, W // 2 + 2, 64), device=dev)
        ops.conv_gemm(gs, pcs, kk, H // 2, W // 2, o)
        if masks is not None:
            others = torch.stack([sum(mk[j] for j in range(K) if j != i) for i in range(K)], 0)
            inp = torch.cat([fr.expand(K, -1, -1, -1), mk, others], 1)
        else:
            inp = fr
        ref = F.conv2d(inp.half().double(), wsel.half().double(), None, stride=2, padding=3)
        assert float((from_halo(o, 64).double() - ref).abs().max()) <= 2e-5 * float(ref.abs().max())


def test_resample_and_layout_fp16(dev):
    n, c, h, w = 2, 64, 60, 108
    a = torch.randn(n, c, h, w, device=dev).half()
    u = torch.randn(n, c, h // 2, w // 2, device=dev).half()
    ah, ar = to_halo(a), torch.zeros((n, h + 2, w + 2, c), device=dev, dtype=H16)
    ops.upsample2x_add(ah, to_halo(u), n, h, w, x_relu=ar)
    ref = a.float() + F.interpolate(u.float(), scale_factor=2, mode="bilinear", align_corners=False)
    got = from_halo(ah, c).float()
    assert bool(((got - ref).abs() <= 2.0 ** -11 * ref.abs() + 1e-6).all())
    assert torch.equal(from_halo(ar, c), from_halo(ah, c).relu())
    # skip variant: x = skip (batch 1) + up2x(up)
    sk = torch.randn(1, c, h, w, device=dev).half()
    xs = torch.zeros((n, h + 2, w + 2, c), device=dev, dtype=H16)
    ops.upsample2x_add(xs, to_halo(u), n, h, w, skip=to_halo(sk))
    ref = sk.float() + F.interpolate(u.float(), scale_factor=2, mode="bilinear", align_corners=False)
    assert bool(((from_halo(xs, c).float() - ref).abs() <= 2.0 ** -11 * ref.abs() + 1e-6).all())
    # layout conversion: fp16 HALO <-> fp32 NCHW
    x = torch.randn(n, c, h, w, device=dev)
    xh = to_halo(x)
    assert torch.equal(ops.halo_to_nchw(xh, n, h, w, c), x.half().float())
    h2 = torch.zeros_like(xh)
    ops.nchw_to_halo(x, h2)
    assert torch.equal(h2, xh)
    # channel-window copies with type conversion (value half of the fp32 key|value map -> fp16 cat map)
    x32 = to_halo(x, dtype=torch.float32)
    d = torch.zeros((n, h + 2, w + 2, 96), device=dev, dtype=H16)
    ops.halo_copy(x32[:1].contiguous(), d, n, h, w, 32, src_coff=16, dst_coff=64, relu=True)
    assert torch.equal(from_halo(d, 96)[:, 64:], x[:1, 16:48].relu().half().expand(n, -1, -1, -1))
    d32 = torch.zeros((n, h + 2, w + 2, 64), device=dev)
    ops.halo_copy(xh, d32, n, h, w, 64)
    assert torch.equal(d32, xh.float())


def test_memory_read_fp16_output(dev):
    g = torch.Generator(device="cpu").manual_seed(5)
    K, T, h, w = 2, 3, 6, 9
    hw = h * w
    bk = torch.randn((K, T * hw, 128), generator=g).to(dev)
    bv = torch.randn((K, T * hw, 512), generator=g).to(dev)
    qk = torch.randn((hw, 128), generator=g).to(dev)
    o32 = torch.zeros((K, h + 2, w + 2, 1024), device=dev)
    o16 = torch.zeros((K, h + 2, w + 2, 1024), device=dev, dtype=H16)
    for algo in (ops.MEMREAD_EXACT_SIMT, ops.MEMREAD_TCGEN05):
        ops.memory_read(bk, bv, T * hw, qk, 20, o32, halo_hw=(h, w), algo=algo)
        ops.memory_read(bk, bv, T * hw, qk, 20, o16, halo_hw=(h, w), algo=algo)
        assert torch.equal(o16, o32.half())
    _lib.poll_kernel_error()


# (n, h, w, cin, cout, ks) the cost model splits when a workspace is attached, per operand type (every other shape
# below must keep the single pass); forced split factors of any shape: tests/test_gpu_conv_plans.py
_SPLITS = {
    torch.float16: {(1, 30, 54, 1024, 512, 3), (1, 30, 54, 1024, 640, 3), (1, 60, 108, 512, 512, 3)},
    torch.float32: {(1, 30, 54, 1024, 512, 3), (1, 30, 54, 256, 256, 3), (1, 30, 54, 1024, 640, 3), (1, 60, 108, 512, 512, 3)},
}


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("n,h,w,cin,cout,ks,relu,res", [
    (1, 30, 54, 1024, 512, 3, False, False),   # decoder.compress conv1 / downsample: 14 row tiles, K = 9216; splits
    (1, 30, 54, 256, 256, 3, True, False),     # layer3 3x3: splits in TF32 only (fp16 keeps BN = 32, S = 1)
    (1, 30, 54, 1024, 256, 1, True, False),    # layer3 1x1 reduce: S = 1 (enough row tiles)
    (2, 30, 54, 256, 1024, 1, True, True),     # layer3 1x1 expand + residual, 2 objects: S = 1
    (1, 30, 54, 1024, 640, 3, False, False),   # key|value projection (cout_pad 640): splits
    (1, 60, 108, 512, 512, 3, False, False),   # 54 row tiles: splits
])
def test_conv_split_k(dev, dtype, n, h, w, cin, cout, ks, relu, res):
    """Split-K path of mivos_conv_gemm as the cost model plans it on this device when a workspace is attached: the
    plan must split the shapes of _SPLITS and keep the single pass (bit-identical to the run without workspace) on the
    others.  Split runs must agree with the single-pass kernel up to fp32 summation order, with an fp64 convolution of
    the same rounded operands, and be repeatable on a reused workspace (fixed summation order)."""
    g = torch.Generator(device="cpu").manual_seed(cin + cout + ks)
    x = torch.randn((n, cin, h, w), generator=g).to(dev)
    wt = (torch.randn((cout, cin, ks, ks), generator=g) / (cin * ks * ks) ** 0.5).to(dev)
    b = torch.randn((cout,), generator=g).to(dev)
    pc = ops.pack_conv(wt, b, device=dev, dtype=dtype)
    xin = to_halo(x, pc.cin_pad, dtype)
    r = torch.randn((n, cout, h, w), generator=g).to(dev) if res else None
    rh = to_halo(r, pc.cout_pad, dtype) if res else None
    ws = ops.split_k_workspace(dev)
    a = _lib.ConvArgs()
    a.n, a.h, a.w, a.taps, a.cin_pad = n, h, w, pc.taps, pc.cin_pad
    a.cout, a.cout_pad = pc.cout, pc.cout_pad
    a.in_f16 = a.out_f16 = int(dtype == torch.float16)
    a.residual = rh.data_ptr() if res else None
    a.splitk_ws, a.splitk_ws_bytes = ws.data_ptr(), ws.numel()
    bn, splits = ctypes.c_int(0), ctypes.c_int(0)
    _lib.check(_lib.load().mivos_conv_plan(ctypes.byref(a), 0, ctypes.byref(bn), ctypes.byref(splits)), "mivos_conv_plan")
    meant_to_split = (n, h, w, cin, cout, ks) in _SPLITS[dtype]
    assert (splits.value >= 2) == meant_to_split, f"planned BN={bn.value} S={splits.value}"
    outs = []
    for use_ws in (None, ws, ws, ws):
        out = torch.full((n, h + 2, w + 2, pc.cout_pad), 7.0, device=dev, dtype=dtype)
        ops.conv_gemm(xin, pc, n, h, w, out, relu=relu, residual=rh, splitk_ws=use_ws)
        outs.append(out)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    assert torch.equal(outs[1], outs[2]) and torch.equal(outs[2], outs[3])  # deterministic reduction order
    if not meant_to_split:
        assert torch.equal(outs[0], outs[1])  # the same single-pass launch with or without a workspace
    if dtype == torch.float16:
        xr, wr = x.half(), wt.half()
    else:  # kind::tf32 truncates the activations; the packed weights are rounded (rna)
        xr, wr = (x.view(torch.int32) & ~0x1FFF).view(torch.float32), ops.round_tf32(wt)
    y = F.conv2d(xr.double(), wr.double(), b.double(), padding=ks // 2)
    if res:
        y = y + r.to(dtype).double()
    y = y.relu() if relu else y
    scale = float(y.abs().max())
    for o in (outs[0], outs[1]):
        got = from_halo(o, cout).double()
        tol = 2e-5 * scale + (2.0 ** -11 * y.abs() if dtype == torch.float16 else 0)
        assert bool(((got - y).abs() <= tol).all())
        assert _border_kept(o)
