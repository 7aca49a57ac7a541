"""GPU: every tile width and forced split-K factor of mivos_conv_gemm, whatever the cost model would pick.

The plan is forced with mivos_conv_tile_override(bn, splits).  Each case is compared against an fp64 convolution of the
same rounded operands (TF32-truncated activations / fp16 activations, the packed weights) with the bound of DESIGN.md
section 6: 2e-5 of the output range, plus one rounding of the result (2^-11 relative) for fp16 or round_tf32 outputs.
Output maps are prefilled with a sentinel that must survive everywhere outside the written window (HALO border,
padded channels, channels outside [out_coff, out_coff + cout)).  The tile widths of one input must give the same
bits: a wgmma accumulates every output element over the same k-block sequence whatever the tile width N is."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402
from test_gpu_zz_batched_ops import pc3_weight_as_conv  # noqa: E402

H16 = torch.float16
SENT = -777.0  # exact in fp16 and fp32
WIDTHS = (32, 64, 128, 256)
# activation type -> (operand dtype, output dtype, round_tf32)
COMBOS = {
    "tf32": (torch.float32, torch.float32, False),
    "tf32_round": (torch.float32, torch.float32, True),
    "fp16": (H16, H16, False),
    "fp16_out32": (H16, torch.float32, False),
}


@pytest.fixture
def force_plan():
    """Force the conv plan; the override is process-global, so it is reset to automatic even when the test fails."""
    lib = _lib.load()

    def force(bn, splits=0):
        _lib.check(lib.mivos_conv_tile_override(bn, splits), "mivos_conv_tile_override")
    yield force
    _lib.check(lib.mivos_conv_tile_override(0, 0), "mivos_conv_tile_override")


def _halo(x, cstride, coff=0, dtype=torch.float32, fill=0.0):
    n, c, h, w = x.shape
    hb = torch.full((n, h + 2, w + 2, cstride), fill, device=x.device, dtype=dtype)
    hb[:, 1:-1, 1:-1, coff:coff + c] = x.permute(0, 2, 3, 1).to(dtype)
    return hb


def _operand(x, dtype):
    """What the tensor core multiplies: fp16 values, or fp32 truncated to TF32."""
    if dtype == H16:
        return x.half().double()
    return (x.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32).double()


def _packed_as_conv(pc):
    """The packed (rounded) weights as an fp64 [cout, cin, k, k] kernel."""
    W = pc.weight.double()
    if pc.taps == 9:
        return W[:, :pc.cout, :pc.cin].reshape(3, 3, pc.cout, pc.cin).permute(2, 3, 0, 1).contiguous()
    return W[0, :pc.cout, :pc.cin].reshape(pc.cout, pc.cin, 1, 1)


def _conv(x_in, pc, n, h, w, odt, *, out_cstride=None, out_coff=0, relu=False, residual=None, res_coff=0,
          dual=False, relu_cstride=None, relu_coff=0, round_tf32=False, ws=None):
    dev = x_in.device
    out = torch.full((n, h + 2, w + 2, out_cstride or pc.cout_pad), SENT, device=dev, dtype=odt)
    out2 = torch.full((n, h + 2, w + 2, relu_cstride or pc.cout_pad), SENT, device=dev, dtype=odt) if dual else None
    ops.conv_gemm(x_in, pc, n, h, w, out, out_coff=out_coff, relu=relu, residual=residual, res_coff=res_coff,
                  out_relu=out2, out_relu_coff=relu_coff, round_tf32=round_tf32, splitk_ws=ws)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    return out, out2


def _window(out, coff, cout):
    m = torch.zeros(out.shape, dtype=torch.bool, device=out.device)
    m[:, 1:-1, 1:-1, coff:coff + cout] = True
    return m


def _check(out, coff, cout, y, rounded, out2=None, coff2=0, what=""):
    """out (HALO, window [coff, coff + cout)) against the fp64 reference y (NCHW); sentinels outside the window."""
    win = _window(out, coff, cout)
    assert bool((out[~win] == SENT).all()), f"{what}: write outside the output window"
    got = out[:, 1:-1, 1:-1, coff:coff + cout].permute(0, 3, 1, 2).double()
    tol = 2e-5 * float(y.abs().max()) + (2.0 ** -11 * y.abs() if rounded else 0.0)
    err = (got - y).abs() - tol
    assert bool((err <= 0).all()), f"{what}: exceeds the fp64 bound by {float(err.max()):.3e}"
    if rounded and out.dtype == torch.float32:
        assert int((out.view(torch.int32)[win] & 0x1FFF).abs().max()) == 0, f"{what}: output not rounded to TF32"
    if out2 is not None:
        win2 = _window(out2, coff2, cout)
        assert bool((out2[~win2] == SENT).all()), f"{what}: ReLU copy written outside its window"
        assert torch.equal(out2[:, 1:-1, 1:-1, coff2:coff2 + cout], out[:, 1:-1, 1:-1, coff:coff + cout].relu()), what


def _layer(seed, n, h, w, cin, cout, ks, dtype, dev):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn((n, cin, h, w), generator=g).to(dev)
    wt = (torch.randn((cout, cin, ks, ks), generator=g) / (cin * ks * ks) ** 0.5).to(dev)
    b = torch.randn((cout,), generator=g).to(dev)
    r = torch.randn((n, cout, h, w), generator=g).to(dev)
    return x, ops.pack_conv(wt, b, device=dev, dtype=dtype), b, r


def _reference(x, pc, b, ks, dtype, odt, relu, r):
    y = F.conv2d(_operand(x, dtype), _packed_as_conv(pc), b.double(), padding=ks // 2)
    if r is not None:
        y = y + r.to(odt).double()
    return y.relu() if relu else y


@pytest.mark.parametrize("combo", list(COMBOS))
@pytest.mark.parametrize("n,h,w,cin,cout,ks,res,relu,dual", [
    pytest.param(1, 120, 216, 64, 64, 3, False, False, False, id="layer1"),
    pytest.param(3, 13, 21, 64, 256, 3, True, True, False, id="batch_tiles_straddle_images"),  # 345 HALO rows per image
    pytest.param(1, 7, 5, 64, 256, 3, False, False, True, id="single_partial_row_tile"),
    pytest.param(2, 30, 54, 128, 256, 1, True, True, True, id="1x1_residual_relu_dual"),
    pytest.param(1, 30, 54, 64, 100, 3, False, True, False, id="ragged_100_of_128"),
    pytest.param(1, 30, 54, 128, 232, 1, True, False, True, id="ragged_232_of_256"),
])
def test_every_tile_width(dev, force_plan, combo, n, h, w, cin, cout, ks, res, relu, dual):
    dtype, odt, rnd = COMBOS[combo]
    x, pc, b, r = _layer(cin * 13 + cout + n, n, h, w, cin, cout, ks, dtype, dev)
    xin = _halo(x, pc.cin_pad, dtype=dtype)
    rh = _halo(r, pc.cout_pad, dtype=odt) if res else None
    y = _reference(x, pc, b, ks, dtype, odt, relu, r if res else None)
    outs = {}
    for bn in WIDTHS:
        if pc.cout_pad % bn:
            continue
        force_plan(bn)
        out, out2 = _conv(xin, pc, n, h, w, odt, relu=relu, residual=rh, dual=dual, round_tf32=rnd)
        _check(out, 0, cout, y, rnd or odt == H16, out2, what=f"BN={bn}")
        outs[bn] = out
    widths = list(outs)
    for bn in widths[1:]:
        assert torch.equal(outs[bn], outs[widths[0]]), f"BN={bn} and BN={widths[0]} differ"


@pytest.mark.parametrize("combo", list(COMBOS))
def test_every_tile_width_s2d_stem(dev, force_plan, combo):
    """The 4-tap space-to-depth stem (mivos_stem_gather_s2d): cout 64, so tile widths 32 and 64."""
    dtype, odt, rnd = COMBOS[combo]
    g = torch.Generator().manual_seed(23)
    C, H, W = 2, 96, 160
    frames = torch.randn((C, 3, H, W), generator=g).to(dev)
    wt = (torch.randn((64, 3, 7, 7), generator=g) / 15).to(dev)
    b = torch.randn((64,), generator=g).to(dev)
    pc = ops.pack_conv(wt, b, stride=2, device=dev, dtype=dtype, stem_s2d=True)
    gm = torch.zeros((C * (H // 2 + 2) * (W // 2 + 2), pc.cin_pad), device=dev, dtype=dtype)
    ops.stem_gather(frames, None, gm, s2d=True)
    y = F.conv2d(_operand(frames, dtype), pc3_weight_as_conv(pc, 3), b.double(), stride=2, padding=3).relu()
    outs = []
    for bn in (32, 64):
        force_plan(bn)
        out, _ = _conv(gm, pc, C, H // 2, W // 2, odt, relu=True, round_tf32=rnd)
        _check(out, 0, 64, y, rnd or odt == H16, what=f"BN={bn}")
        outs.append(out)
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("combo", ["tf32", "fp16"])
def test_output_window_every_tile_width(dev, force_plan, combo):
    """out_coff / out_relu_coff / res_coff windows of maps wider than cout_pad: how the S2M ASPP concat map
    (five 256-channel branches side by side) is written."""
    dtype, odt, _ = COMBOS[combo]
    n, h, w, cin, cout = 2, 17, 29, 128, 256
    x, pc, b, r = _layer(99, n, h, w, cin, cout, 3, dtype, dev)
    xin = _halo(x, pc.cin_pad, dtype=dtype)
    rh = _halo(r, 768, coff=384, dtype=odt, fill=5.0)  # channels outside the residual window must not be read
    y = _reference(x, pc, b, 3, dtype, odt, False, r)
    outs = []
    for bn in WIDTHS:
        force_plan(bn)
        out, out2 = _conv(xin, pc, n, h, w, odt, out_cstride=1280, out_coff=512, residual=rh, res_coff=384,
                          dual=True, relu_cstride=640, relu_coff=256)
        _check(out, 512, cout, y, odt == H16, out2, coff2=256, what=f"BN={bn}")
        outs.append((out, out2))
    for o, o2 in outs[1:]:
        assert torch.equal(o, outs[0][0]) and torch.equal(o2, outs[0][1])


@pytest.mark.parametrize("combo", ["tf32", "fp16"])
def test_forced_split_k_factors(dev, force_plan, combo):
    """decoder.compress (1, 30, 54, 1024 -> 512, 3x3) under S = 2, 3, 5, 7, 8 (144 fp16 / 288 TF32 k-blocks: 5 and 7
    give K ranges of unequal length), each with another tile width; repeat runs over the reused workspace are
    bit-identical (the second pass sums the partials in split order)."""
    dtype, odt, _ = COMBOS[combo]
    n, h, w, cin, cout = 1, 30, 54, 1024, 512
    x, pc, b, _ = _layer(7, n, h, w, cin, cout, 3, dtype, dev)
    xin = _halo(x, pc.cin_pad, dtype=dtype)
    y = _reference(x, pc, b, 3, dtype, odt, False, None)
    ws = ops.split_k_workspace(dev)
    for splits, bn in ((2, 256), (3, 128), (5, 64), (7, 128), (8, 32)):
        force_plan(bn, splits)
        out, _ = _conv(xin, pc, n, h, w, odt, ws=ws)
        _check(out, 0, cout, y, odt == H16, what=f"S={splits} BN={bn}")
        again, _ = _conv(xin, pc, n, h, w, odt, ws=ws)
        assert torch.equal(out, again), f"S={splits} BN={bn}: not repeatable"


@pytest.mark.parametrize("combo", ["tf32_round", "fp16"])
def test_forced_split_k_epilogue_forms(dev, force_plan, combo):
    """The second pass of split-K (splitk_epilogue_kernel) with a ragged channel tail, residual, ReLU copy,
    round_tf32 and output windows.  cout 498 of 512: whole 4-channel pieces past cout are skipped and the last piece
    holds 2 real channels."""
    dtype, odt, rnd = COMBOS[combo]
    n, h, w, cin, cout = 1, 30, 54, 512, 498
    x, pc, b, r = _layer(11, n, h, w, cin, cout, 3, dtype, dev)
    xin = _halo(x, pc.cin_pad, dtype=dtype)
    rh = _halo(r, 1024, coff=256, dtype=odt, fill=5.0)
    y = _reference(x, pc, b, 3, dtype, odt, False, r)
    ws = ops.split_k_workspace(dev)
    for splits, bn in ((3, 128), (5, 256)):
        force_plan(bn, splits)
        kw = dict(out_cstride=1024, out_coff=512, residual=rh, res_coff=256, dual=True, relu_cstride=768,
                  relu_coff=128, round_tf32=rnd, ws=ws)
        out, out2 = _conv(xin, pc, n, h, w, odt, **kw)
        _check(out, 512, cout, y, True, out2, coff2=128, what=f"S={splits} BN={bn}")
        again, again2 = _conv(xin, pc, n, h, w, odt, **kw)
        assert torch.equal(out, again) and torch.equal(out2, again2), f"S={splits} BN={bn}: not repeatable"
