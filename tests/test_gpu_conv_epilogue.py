"""GPU: the convolution epilogue's bulk copies - residual rows prefetched into the staging tile, output rows stored
from it - at the shapes where they are easiest to get wrong.

Each case is compared against an fp64 convolution of the rounded operands with the bound of test_gpu_conv_plans.py,
and every admissible tile width must give the same bits.  Output maps are prefilled with a sentinel that must survive
in the HALO border and past cout; the residual's border rows and the channels outside its window hold NaN, so a
read of any of them shows up as a NaN in the output."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402
from test_gpu_conv_plans import COMBOS, SENT, WIDTHS, _check, _conv, _halo, _layer, _reference, force_plan  # noqa: E402,F401

NAN = float("nan")


def _every_width(dev, force_plan, combo, n, h, w, cin, cout, ks, *, seed, relu=True, res_cstride=None, res_coff=0,
                 out_cstride=None, out_coff=0, relu_cstride=None, relu_coff=0):
    """Residual + ReLU copy at every tile width; returns the outputs of the first width."""
    dtype, odt, rnd = COMBOS[combo]
    x, pc, b, r = _layer(seed, n, h, w, cin, cout, ks, dtype, dev)
    xin = _halo(x, pc.cin_pad, dtype=dtype)
    rh = _halo(r, res_cstride or pc.cout_pad, coff=res_coff, dtype=odt, fill=NAN)
    y = _reference(x, pc, b, ks, dtype, odt, relu, r)
    outs = {}
    for bn in WIDTHS:
        if pc.cout_pad % bn:
            continue
        force_plan(bn)
        out, out2 = _conv(xin, pc, n, h, w, odt, out_cstride=out_cstride, out_coff=out_coff, relu=relu, residual=rh,
                          res_coff=res_coff, dual=True, relu_cstride=relu_cstride, relu_coff=relu_coff, round_tf32=rnd)
        _check(out, out_coff, cout, y, rnd or odt == torch.float16, out2, coff2=relu_coff, what=f"BN={bn}")
        outs[bn] = (out, out2)
    first = next(iter(outs))
    for bn, (o, o2) in outs.items():
        assert torch.equal(o, outs[first][0]) and torch.equal(o2, outs[first][1]), f"BN={bn} and BN={first} differ"


@pytest.mark.parametrize("combo", list(COMBOS))
@pytest.mark.parametrize("n,h,w,cin,ks", [
    pytest.param(2, 30, 54, 64, 1, id="1x1_64_few_kblocks"),  # residual loaded with the first operands
    pytest.param(1, 30, 54, 512, 3, id="3x3_512_long_loop"),  # residual waits for the stages under it to drain
])
def test_residual_prefetch(dev, force_plan, combo, n, h, w, cin, ks):
    _every_width(dev, force_plan, combo, n, h, w, cin, 256, ks, seed=cin + ks)


@pytest.mark.parametrize("combo", ["tf32", "fp16"])
@pytest.mark.parametrize("w", [1, 2, 5])
def test_tiles_straddle_rows_and_images(dev, force_plan, combo, w):
    """n = 3 maps only 1, 2 or 5 pixels wide: a 128-row tile spans many image rows, several images and their
    borders, and the last tile is partial."""
    _every_width(dev, force_plan, combo, 3, 37, w, 64, 64, 3, seed=w)


@pytest.mark.parametrize("combo", list(COMBOS))
@pytest.mark.parametrize("cout", [1, 36, 100, 250])
def test_ragged_channels_in_windows(dev, force_plan, combo, cout):
    """Row segments whose bytes are not a multiple of 16 (bulk head + element-wise tail), written into channel
    windows of wider maps, with the residual read from a window of a NaN-filled map."""
    _every_width(dev, force_plan, combo, 2, 13, 21, 64, cout, 1 if cout % 2 else 3, seed=cout,
                 res_cstride=384, res_coff=64, out_cstride=320, out_coff=32, relu_cstride=288, relu_coff=16)


@pytest.mark.parametrize("combo", ["tf32", "fp16"])
def test_chained_convs_in_graph(dev, combo):
    """Two PDL-chained convs, the second reading the first's bulk-stored output at once as operand and residual:
    replays of a CUDA graph give the bits of eager launches with a synchronise between them."""
    dtype, odt, _ = COMBOS[combo]
    n, h, w = 2, 60, 108
    x, pc1, _, r = _layer(5, n, h, w, 64, 256, 1, dtype, dev)
    _, pc2, _, _ = _layer(6, n, h, w, 256, 256, 1, dtype, dev)
    xin = _halo(x, pc1.cin_pad, dtype=dtype)
    rh = _halo(r, 256, dtype=odt)
    y1 = torch.zeros((n, h + 2, w + 2, 256), device=dev, dtype=dtype)
    y2 = torch.full((n, h + 2, w + 2, 256), SENT, device=dev, dtype=dtype)

    def run(sync):
        ops.conv_gemm(xin, pc1, n, h, w, y1, relu=True, residual=rh)
        if sync:
            torch.cuda.synchronize()
        ops.conv_gemm(y1, pc2, n, h, w, y2, relu=True, residual=y1)

    run(True)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    want1, want2 = y1.clone(), y2.clone()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run(False)
    for _ in range(2):
        y1.zero_()
        y2.fill_(SENT)
        g.replay()
        torch.cuda.synchronize()
        _lib.poll_kernel_error()
        assert torch.equal(y1, want1) and torch.equal(y2, want2)
