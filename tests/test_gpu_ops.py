"""GPU: every C-ABI kernel against a plain PyTorch reference of the same op on the same seeded
inputs.  Convolutions run TF32 (operands truncated to 10-bit mantissa by the tensor core, fp32
accumulate): they are compared (a) against an fp64 convolution of the TF32-truncated operands —
tolerance 2e-5 of the output range, i.e. the kernel is exact up to accumulation order — and
(b) against the fp32 op with the TF32 tolerance 2e-3.  Integer/byte/index work is bit-exact."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402


def to_halo(x, cpad=None):
    n, c, h, w = x.shape
    hb = torch.zeros((n, h + 2, w + 2, cpad or c), device=x.device, dtype=torch.float32)
    hb[:, 1:-1, 1:-1, :c] = x.permute(0, 2, 3, 1)
    return hb


def from_halo(hb, c):
    return hb[:, 1:-1, 1:-1, :c].permute(0, 3, 1, 2).contiguous()


def trunc_tf32(x):
    return (x.view(torch.int32) & ~0x1FFF).view(torch.float32)


@pytest.mark.parametrize("n,h,w,cin,cout,ks,relu,res,dual", [
    (1, 30, 54, 64, 64, 3, False, False, False),     # 28 row tiles of BN=32 (the plan at 132 SMs)
    (1, 30, 54, 32, 1, 3, False, False, False),      # decoder.pred shape: one real output channel
    (1, 30, 54, 256, 64, 1, True, False, False),     # bottleneck 1x1 + relu
    (2, 60, 108, 128, 128, 3, True, True, False),    # batch 2, residual + relu
    (1, 120, 216, 256, 256, 3, False, False, True),  # 208 tiles of BN=256, dual (raw + relu) output
    (1, 30, 54, 1024, 640, 3, False, False, False),  # fused key|value projection
    (1, 7, 5, 32, 32, 3, False, False, False),       # tiny ragged map (single partial M tile)
    (1, 120, 216, 64, 128, 1, True, True, True),     # 208 tiles of BN=128, residual + dual
    (1, 120, 216, 64, 64, 3, True, False, False),    # 208 tiles of BN=64 (every tile width: test_gpu_conv_plans.py)
    (1, 240, 432, 32, 20, 3, False, False, False),   # 821 tiles of BN=32, ragged channel tail (20 of 32)
])
def test_conv_gemm(dev, n, h, w, cin, cout, ks, relu, res, dual):
    g = torch.Generator(device="cpu").manual_seed(cin * 7 + cout)
    x = torch.randn((n, cin, h, w), generator=g).to(dev)
    wt = (torch.randn((cout, cin, ks, ks), generator=g) / (cin * ks * ks) ** 0.5).to(dev)
    b = torch.randn((cout,), generator=g).to(dev)
    pc = ops.pack_conv(wt, b, device=dev)
    xin = to_halo(x, pc.cin_pad)
    out = torch.full((n, h + 2, w + 2, pc.cout_pad), 7.0, device=dev)  # sentinel: halo/pad lanes must stay 7
    r = torch.randn((n, cout, h, w), generator=g).to(dev) if res else None
    out2 = torch.zeros_like(out) if dual else None
    ops.conv_gemm(xin, pc, n, h, w, out, relu=relu, residual=to_halo(r, pc.cout_pad) if res else None, out_relu=out2)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    got = from_halo(out, cout).double()

    def ref(f):
        y = F.conv2d(f(x).double(), ops.round_tf32(wt).double(), b.double(), padding=ks // 2)
        if res:
            y = y + r.double()
        return y.relu() if relu else y
    exact, fp32 = ref(trunc_tf32), ref(lambda t: t)
    scale = float(fp32.abs().max())
    assert float((got - exact).abs().max()) <= 2e-5 * scale
    assert float((got - fp32).abs().max()) <= 2e-3 * scale
    assert bool((out[:, 0] == 7).all() and (out[:, -1] == 7).all() and (out[:, :, 0] == 7).all() and (out[:, :, -1] == 7).all())
    if pc.cout_pad > cout:
        assert bool((out[:, 1:-1, 1:-1, cout:] == 7).all())
    if dual:
        assert torch.equal(from_halo(out2, cout), from_halo(out, cout).relu())


def test_conv_round_tf32_flag(dev):
    x = torch.randn((1, 32, 8, 8), device=dev)
    wt = torch.randn((32, 32, 3, 3), device=dev) / 17
    pc = ops.pack_conv(wt, None, device=dev)
    out = torch.zeros((1, 10, 10, 32), device=dev)
    ops.conv_gemm(to_halo(x), pc, 1, 8, 8, out, round_tf32=True)
    assert int((out.view(torch.int32) & 0x1FFF).abs().max()) == 0


def test_strided_and_stem_gathers(dev):
    n, c, h, w = 2, 64, 60, 108
    x = torch.randn(n, c, h, w, device=dev).relu()
    xh = to_halo(x)
    out = torch.zeros((n, h // 2 + 2, w // 2 + 2, c), device=dev)
    ops.maxpool3x3s2(xh, n, h, w, out)
    assert torch.equal(from_halo(out, c), F.max_pool2d(x, 3, 2, 1))
    for ks, cout in ((3, 96), (1, 128)):
        wt = torch.randn(cout, c, ks, ks, device=dev) / (c * ks * ks) ** 0.5
        b = torch.randn(cout, device=dev)
        pc = ops.pack_conv(wt, b, stride=2, im2col=True, device=dev)
        g = torch.zeros((n * (h // 2 + 2) * (w // 2 + 2), pc.cin_pad), device=dev)
        ops.gather_s2(xh, n, h, w, c, ks, g)
        o = torch.zeros((n, h // 2 + 2, w // 2 + 2, pc.cout_pad), device=dev)
        ops.conv_gemm(g, pc, n, h // 2, w // 2, o)
        ref = F.conv2d(x.double(), wt.double(), b.double(), stride=2, padding=ks // 2)
        assert float((from_halo(o, cout).double() - ref).abs().max()) <= 2e-3 * float(ref.abs().max())
    H, W, K = 96, 160, 3
    fr = torch.randn(1, 3, H, W, device=dev)
    mk = torch.rand(K, 1, H, W, device=dev)
    ws = torch.randn(64, 5, 7, 7, device=dev) / 15
    for masks, wsel, kk in ((mk, ws, K), (None, ws[:, :3].contiguous(), 1)):
        pcs = ops.pack_conv(wsel, None, stride=2, im2col=True, device=dev)
        gs = torch.zeros((kk * (H // 2 + 2) * (W // 2 + 2), pcs.cin_pad), device=dev)
        ops.stem_gather(fr, masks, gs)
        o = torch.zeros((kk, H // 2 + 2, W // 2 + 2, 64), device=dev)
        ops.conv_gemm(gs, pcs, kk, H // 2, W // 2, o)
        if masks is not None:
            others = torch.stack([sum(mk[j] for j in range(K) if j != i) for i in range(K)], 0)
            inp = torch.cat([fr.expand(K, -1, -1, -1), mk, others], 1)
        else:
            inp = fr
        ref = F.conv2d(inp.double(), wsel.double(), None, stride=2, padding=3)
        assert float((from_halo(o, 64).double() - ref).abs().max()) <= 2e-3 * float(ref.abs().max())


def test_resample_layout_aggregate_argmax(dev):
    n, c, h, w = 2, 64, 60, 108
    a = torch.randn(n, c, h, w, device=dev)
    u = torch.randn(n, c, h // 2, w // 2, device=dev)
    ah, ar = to_halo(a), torch.zeros((n, h + 2, w + 2, c), device=dev)
    ops.upsample2x_add(ah, to_halo(u), n, h, w, x_relu=ar)
    ref = a + F.interpolate(u, scale_factor=2, mode="bilinear", align_corners=False)
    assert float((from_halo(ah, c) - ref).abs().max()) <= 2e-6 and float((from_halo(ar, c) - ref.relu()).abs().max()) <= 2e-6
    x = torch.randn(n, c, h, w, device=dev)
    xh = to_halo(x)
    assert torch.equal(ops.halo_to_nchw(xh, n, h, w, c), x)
    h2 = torch.zeros_like(xh)
    ops.nchw_to_halo(x, h2)
    assert torch.equal(h2, xh)
    px = torch.empty((n, h * w, 16), device=dev)
    ops.halo_to_pixels(xh, n, h, w, 8, 16, px)
    assert torch.equal(px, x[:, 8:24].reshape(n, 16, h * w).transpose(1, 2))
    d = torch.zeros((n, h + 2, w + 2, 96), device=dev)
    ops.halo_copy(xh[:1].contiguous(), d, n, h, w, 32, src_coff=16, dst_coff=64, relu=True)
    assert torch.equal(from_halo(d, 96)[:, 64:], x[:1, 16:48].relu().expand(n, -1, -1, -1))
    k, h4, w4 = 3, 24, 40
    lg = torch.randn(k, 1, h4, w4, device=dev) * 3
    raw, prob = ops.upsample4x_sigmoid_aggregate(to_halo(lg, 32), k, h4, w4, want_raw=True)
    r = torch.sigmoid(F.interpolate(lg, scale_factor=4, mode="bilinear", align_corners=False))
    assert float((raw - r).abs().max()) <= 1e-6
    newp = torch.cat([torch.prod(1 - r, dim=0, keepdim=True), r], 0).clamp(1e-7, 1 - 1e-7)
    lgt = torch.log(newp / (1 - newp))
    assert float((prob - F.softmax(lgt, dim=0)).abs().max()) <= 1e-6
    assert float((ops.aggregate_wbg(r, keep_bg=True) - F.softmax(lgt, dim=0)).abs().max()) <= 1e-6
    assert float((ops.aggregate_wbg(r, keep_bg=False, hard=True) - F.softmax(lgt * 1000, dim=0)[1:]).abs().max()) <= 1e-6
    sb = torch.cat([torch.full_like(r[:1], 0.5), r], 0).clamp(1e-7, 1 - 1e-7)
    assert float((ops.aggregate_wbg(r, keep_bg=True, const_bg=True) - F.softmax(torch.log(sb / (1 - sb)), dim=0)).abs().max()) <= 1e-6
    T = 4
    pr = torch.rand(k + 1, T, 1, 48, 64, device=dev)
    pr[1, :, :, :5] = pr[0, :, :, :5]  # exact ties: the first maximum wins, like torch.argmax on CPU
    mp = torch.zeros((T, 1, 48, 64), dtype=torch.uint8, device=dev)
    mo = torch.zeros((T, 44, 60), dtype=torch.uint8, device=dev)
    ops.argmax_unpad(pr, (2, 2, 2, 2), 44, 60, mp, mo)
    ref = torch.argmax(pr.cpu(), 0).to(torch.uint8).to(dev)
    assert torch.equal(mp, ref) and torch.equal(mo, ref[:, 0, 2:-2, 2:-2])
    assert torch.equal(ops.pad2d(pr, (3, 4, 1, 2)), F.pad(pr, (3, 4, 1, 2)))


def test_attention_map(dev):
    h16, w16 = 12, 20
    hw = h16 * w16
    mk = torch.randn(1, 128, 1, h16, w16, device=dev)
    qk = torch.randn(1, 128, h16, w16, device=dev)
    pos = torch.rand(1, 1, h16 * 16, w16 * 16, device=dev)
    neg = torch.rand(1, 1, h16 * 16, w16 * 16, device=dev)
    out = ops.attention_map(mk.reshape(128, hw).t().contiguous(), qk.reshape(128, hw).t().contiguous(), h16, w16, pos, neg)
    Wm = F.softmax(torch.bmm(mk.reshape(1, 128, hw).transpose(1, 2).double(), (qk.reshape(1, 128, hw) / 128 ** 0.5).double()), dim=1)
    pm = F.interpolate(pos, size=(h16, w16), mode="area").view(1, 1, hw).double() @ Wm
    nm = F.interpolate(neg, size=(h16, w16), mode="area").view(1, 1, hw).double() @ Wm
    ref = F.interpolate(torch.cat([pm, nm], 1).reshape(1, 2, h16, w16), mode="bilinear", size=(h16 * 16, w16 * 16), align_corners=False)
    assert float((out.double() - ref).abs().max()) <= 5e-6
