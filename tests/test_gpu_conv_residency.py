"""GPU: the two-CTAs-per-SM class of mivos_conv_gemm gives the bits of the one-CTA class.

Residency changes where a tile runs, not what it computes: each tile issues the same wgmmas over the same k-block
sequence, so every output element must be bit-identical to the one-CTA kernel's at the same tile width and split-K
factor.  Covered: BN 32 and 64 (the two-CTA class), TF32 and fp16 operands, 1, 4 (space-to-depth stem) and 9 taps,
plain / +residual / +ReLU copy / split-K 2 and 3, at ragged shapes (partial row tiles, cout below cout_pad).  Every
launch of a two-CTA kernel first checks with cudaOccupancyMaxActiveBlocksPerMultiprocessor that it reaches two CTAs
per SM and fails otherwise, so each passing case also shows that query returned 2."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402
from test_gpu_conv_plans import COMBOS, SENT, _conv, _halo, _layer, _window  # noqa: E402


@pytest.fixture
def force():
    """Force tile width, split-K factor and residency; both overrides are process-global, so they are reset to
    automatic even when the test fails."""
    lib = _lib.load()

    def set_plan(bn, splits, ctas):
        _lib.check(lib.mivos_conv_residency_override(0), "mivos_conv_residency_override")
        _lib.check(lib.mivos_conv_tile_override(bn, splits), "mivos_conv_tile_override")
        _lib.check(lib.mivos_conv_residency_override(ctas), "mivos_conv_residency_override")
    yield set_plan
    _lib.check(lib.mivos_conv_residency_override(0), "mivos_conv_residency_override")
    _lib.check(lib.mivos_conv_tile_override(0, 0), "mivos_conv_tile_override")


def _operands(taps, dtype, odt, dev):
    """(input map, packed conv, n, h, w, HALO residual) of a ragged layer with `taps` taps."""
    if taps == 4:  # the space-to-depth stem: 7x7/2 over 3 channels, gathered into 4 vertical taps
        g = torch.Generator().manual_seed(41)
        n, H, W = 2, 70, 102  # 35 x 51 output pixels: partial last row tile
        frames = torch.randn((n, 3, H, W), generator=g).to(dev)
        wt = (torch.randn((64, 3, 7, 7), generator=g) / 15).to(dev)
        b = torch.randn((64,), generator=g).to(dev)
        pc = ops.pack_conv(wt, b, stride=2, device=dev, dtype=dtype, stem_s2d=True)
        h, w = H // 2, W // 2
        xin = torch.zeros((n * (h + 2) * (w + 2), pc.cin_pad), device=dev, dtype=dtype)
        ops.stem_gather(frames, None, xin, s2d=True)
        r = torch.randn((n, 64, h, w), generator=g).to(dev)
        return xin, pc, n, h, w, _halo(r, pc.cout_pad, dtype=odt)
    n, h, w, cin, cout = (3, 13, 21, 192, 100) if taps == 9 else (2, 29, 37, 320, 120)
    x, pc, _, r = _layer(cin + cout + taps, n, h, w, cin, cout, 3 if taps == 9 else 1, dtype, dev)
    return _halo(x, pc.cin_pad, dtype=dtype), pc, n, h, w, _halo(r, pc.cout_pad, dtype=odt)


@pytest.mark.parametrize("combo", ["tf32", "fp16"])
@pytest.mark.parametrize("taps", [1, 4, 9])
@pytest.mark.parametrize("bn", [32, 64])
@pytest.mark.parametrize("form", ["plain", "residual", "out_relu", "split2", "split3"])
def test_two_ctas_per_sm_give_the_one_cta_bits(dev, force, combo, taps, bn, form):
    dtype, odt, _ = COMBOS[combo]
    xin, pc, n, h, w, rh = _operands(taps, dtype, odt, dev)
    splits = {"split2": 2, "split3": 3}.get(form, 0)
    kw = dict(relu=form != "out_relu", residual=rh if form in ("residual", "split2") else None,
              dual=form in ("out_relu", "split3"), ws=ops.split_k_workspace(dev) if splits else None)
    outs = {}
    for ctas in (1, 2):
        force(bn, splits, ctas)
        outs[ctas] = _conv(xin, pc, n, h, w, odt, **kw)
    (o1, r1), (o2, r2) = outs[1], outs[2]
    win = _window(o2, 0, pc.cout)
    assert bool((o2[~win] == SENT).all()), "the two-CTA kernel wrote a HALO border row or a padded channel"
    assert bool((o1[win] != SENT).all()), "the one-CTA kernel left part of the output window unwritten"
    assert torch.equal(o2, o1), "two CTAs per SM and one CTA per SM differ"
    if kw["dual"]:
        assert torch.equal(r2, r1), "the ReLU copies differ"


def test_halo_border_rows_stay_zero_under_two_ctas(dev, force):
    """A map whose HALO border is zero (as every activation map the networks keep) still has a zero border after
    a two-CTA launch with a residual and a ReLU copy: the border rows are never written."""
    xin, pc, n, h, w, rh = _operands(9, torch.float16, torch.float16, dev)
    force(64, 0, 2)
    out = torch.zeros((n, h + 2, w + 2, pc.cout_pad), device=dev, dtype=torch.float16)
    out2 = torch.zeros_like(out)
    ops.conv_gemm(xin, pc, n, h, w, out, relu=True, residual=rh, out_relu=out2)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    for o in (out, out2):
        border = torch.ones(o.shape[:3], dtype=torch.bool, device=dev)
        border[:, 1:-1, 1:-1] = False
        assert int(torch.count_nonzero(o[border])) == 0
        assert int(torch.count_nonzero(o[:, 1:-1, 1:-1, :pc.cout])) > 0


def test_planned_residency_runs_and_matches_one_cta(dev):
    """The layers the planner gives two CTAs per SM at 132 SMs (the layer1 maps of a lock-step batch of four clips)
    run under the automatic plan and give the bits of the forced one-CTA plan."""
    lib = _lib.load()
    n, h, w, cin, cout = 4, 120, 216, 64, 64
    x, pc, _, _ = _layer(5, n, h, w, cin, cout, 3, torch.float16, dev)
    xin = _halo(x, pc.cin_pad, dtype=torch.float16)
    out = torch.empty((n, h + 2, w + 2, pc.cout_pad), device=dev, dtype=torch.float16)
    a = ops.conv_args(xin, pc, n, h, w, out, relu=True)
    ctas = C.c_int(0)
    _lib.check(lib.mivos_conv_plan_residency(C.byref(a), 0, C.byref(ctas)), "mivos_conv_plan_residency")
    assert ctas.value == 2
    auto, _ = _conv(xin, pc, n, h, w, torch.float16, relu=True)
    try:
        _lib.check(lib.mivos_conv_residency_override(1), "mivos_conv_residency_override")
        one, _ = _conv(xin, pc, n, h, w, torch.float16, relu=True)
    finally:
        _lib.check(lib.mivos_conv_residency_override(0), "mivos_conv_residency_override")
    assert torch.equal(auto, one)
