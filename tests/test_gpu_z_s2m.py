"""GPU: the S2M operators (csrc/halo_ops.cu, csrc/elementwise.cu) against plain float64 statements of the same
operations, and the S2M network and controller against the vectors the UNMODIFIED reference produced
(tests/golden/s2m_*.npz).

The operator tests follow tests/test_gpu_ops_ragged.py: every reference is computed from the operands the kernel saw
(fp16-rounded for fp16 maps); the dilated gather is bit-exact; outputs are pre-filled with a sentinel that must
survive outside the written window; inputs the kernel must not read (HALO borders, channels outside the window) hold
NaN.  The arithmetic kernels get elementwise bounds derived from their fp32 operations (u = 2^-24), and every check
prints its largest err/bound ratio (run with -s):
  * halo_avgpool_broadcast: each of 8 pixel groups sums its pixels sequentially, the 8 partials are added, the sum is
    multiplied by fl(1/hw): |m - mu| <= ((ceil(hw/8) + 7) u sum|x|) / hw + 2u |mu|;
  * upsample_bilinear, halo_upsample_to_plane: 5u sum|w v| where the scale in/out is a power of two (exact weights),
    6u sum|w v| elsewhere (1 - l rounds too), plus dsrc D per axis: fl(in/out) and the source coordinate put the
    sample at most dsrc <= 3u (in + 1) off, and the interpolant moves by at most D (the largest difference of
    neighbouring source values along that axis) per unit; through the sigmoid p(1-p) err + p(2u + 4u(1-p));
  * fp16 maps round the result once more: 2^-11 |ref| (2^-25 absolute below the normal range).
Network outputs carry the conv tolerances of DESIGN.md §6 (fp16 / TF32 operands, fp32 accumulation)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402
from test_gpu_ops_ragged import H16, NAN, SENT, U, VEC, _check, _halo, _round16  # noqa: E402
from op_references import avgpool_reference, bilinear_reference  # noqa: E402

DT = {"fp16": torch.float16, "tf32": torch.float32}


def to_halo(x, cpad=None, dtype=torch.float32):
    n, c, h, w = x.shape
    hb = torch.zeros((n, h + 2, w + 2, cpad or c), device=x.device, dtype=dtype)
    hb[:, 1:-1, 1:-1, :c] = x.permute(0, 2, 3, 1).to(dtype)
    return hb


def _sync():
    torch.cuda.synchronize()
    _lib.poll_kernel_error()


def _outside(t, n, h, w, coff, c):
    """Mask of everything but the interior pixels of channels [coff, coff + c) of a HALO map."""
    m = torch.ones(t.shape, dtype=torch.bool, device=t.device)
    m[:, 1:h + 1, 1:w + 1, coff:coff + c] = False
    return m


# ------------------------------------------------------------------------------------------ dilated gather
@pytest.mark.parametrize("dtype", [torch.float32, H16])
@pytest.mark.parametrize("dil", [1, 2, 6, 12, 18])
def test_gather_dilated(dev, dtype, dil):
    """out[r, (ky*3 + kx)*c + ci] = x[y + (ky-1) d, x + (kx-1) d, ci] (zero outside the map): F.unfold(dilation=d,
    padding=d) reordered to (ky, kx, c).  Three images of different content; a d x d map, where only the centre tap
    is live; a (2d + 3) x (d + 5) map, on which dilation d + 1 reads other pixels; c of one 16-byte vector and a c
    that is not a multiple of 32.  The input holds NaN in its border and in one vector of channels past c; the output
    has one vector of columns past 9c that must keep the sentinel, and its HALO border rows are zero rows."""
    v = VEC[dtype]
    g = torch.Generator().manual_seed(dil)
    for n, h, w, c in ((3, 9, 13, 40 if dtype == torch.float32 else 72), (1, dil, dil, v), (2, 5, 3, v),
                       (2, 2 * dil + 3, dil + 5, v)):
        x = torch.randn(n, c, h, w, generator=g).to(dtype).to(dev)
        src = _halo(x, c + v, fill=NAN, dtype=dtype)
        got = torch.full((n, h + 2, w + 2, 9 * c + v), SENT, dtype=dtype, device=dev)
        ops.gather_dilated(src, n, h, w, c, dil, got)
        _sync()
        cols = F.unfold(x.double(), 3, dilation=dil, padding=dil)  # [n, c*9, h*w], (c, ky, kx) order
        cols = cols.reshape(n, c, 9, h, w).permute(0, 3, 4, 2, 1).reshape(n, h, w, 9 * c)
        exp = torch.full_like(got, SENT)
        exp[..., :9 * c] = 0
        exp[:, 1:-1, 1:-1, :9 * c] = cols.to(dtype)
        assert torch.equal(got, exp), f"gather_dilated d={dil} {n}x{h}x{w} c={c}"


# ------------------------------------------------------------------------------------------ pooled broadcast
# (n, h, w, c, in_coff, out_coff, spread of the per-image offsets, common offset)
AVGPOOL_CASES = [
    (2, 1, 1, None, 0, 0, 0.0, 0.0),      # hw = 1
    (1, 1, 5, None, 0, 0, 0.0, 0.0),      # hw = 5: three of the 8 pixel groups idle
    (1, 45, 80, None, 0, 0, 0.0, 0.0),    # the 1/16 map of 720p: 3600 pixels
    (1, 6, 8, 2048, 1, 2, 0.0, 0.0),      # the 2048-channel ASPP input, both channel windows offset (in vectors)
    (3, 5, 7, None, 1, 0, 10.0, 0.0),     # per-image offsets: mixing images shows
    (1, 9, 13, None, 0, 1, 0.0, 1000.0),  # mean 1000, spread 1
]


@pytest.mark.parametrize("dtype", [torch.float32, H16])
@pytest.mark.parametrize("case", range(len(AVGPOOL_CASES)))
def test_avgpool_broadcast(dev, dtype, case):
    n, h, w, c, in_v, out_v, spread, offset = AVGPOOL_CASES[case]
    v = VEC[dtype]
    c = c or (40 if dtype == torch.float32 else 8)  # 10 vectors / 1 vector: neither fills the 32 lanes of a CTA
    in_coff, out_coff = in_v * v, out_v * v
    g = torch.Generator().manual_seed(case)
    base = offset + spread * torch.arange(n, dtype=torch.float32).reshape(n, 1, 1, 1)
    x = (torch.randn(n, c, h, w, generator=g) + base).to(dtype).to(dev)
    src = _halo(x, in_coff + c + v, in_coff, fill=NAN, dtype=dtype)
    out = torch.full((n, h + 2, w + 2, out_coff + c + v), SENT, dtype=dtype, device=dev)
    ops.halo_avgpool_broadcast(src, n, h, w, c, out, in_coff=in_coff, out_coff=out_coff)
    _sync()
    mu, bound = avgpool_reference(x)
    win = out[:, 1:-1, 1:-1, out_coff:out_coff + c]
    assert bool((win == win[:, :1, :1]).all()), "the mean is not the same at every pixel"
    _check(f"avgpool {dtype} n={n} {h}x{w} c={c}", win[:, 0, 0], mu, _round16(bound, mu, dtype))
    assert bool((out[_outside(out, n, h, w, out_coff, c)] == SENT).all()), "written outside the window"


# ------------------------------------------------------------------------------------------ bilinear resizes
# (n, hs, ws, h, w, c (None: a ragged count), src_coff, dst_coff)
RESIZE_CASES = [
    (1, 45, 80, 180, 320, 256, 1, 48),  # x4, the S2M head at 720p: ASPP output into the 304-channel concat map
    (2, 7, 5, 10, 13, None, 0, 0),
    (1, 13, 9, 5, 4, None, 1, 2),       # downsampling
    (3, 1, 1, 6, 8, None, 0, 1),
    (1, 6, 8, 1, 1, None, 2, 0),
]


@pytest.mark.parametrize("dtype", [torch.float32, H16])
@pytest.mark.parametrize("case", range(len(RESIZE_CASES)))
def test_upsample_bilinear_window(dev, dtype, case):
    n, hs, ws, h, w, c, s_v, d_v = RESIZE_CASES[case]
    v = VEC[dtype]
    c = c or (40 if dtype == torch.float32 else 72)
    s_coff = s_v * v
    d_coff = 48 if d_v == 48 else d_v * v
    x = (torch.randn(n, c, hs, ws, generator=torch.Generator().manual_seed(case)) * 3).to(dtype).to(dev)
    src = _halo(x, s_coff + c + v, s_coff, fill=NAN, dtype=dtype)
    out = torch.full((n, h + 2, w + 2, d_coff + c + v), SENT, dtype=dtype, device=dev)
    ops.upsample_bilinear(src, n, hs, ws, out, h, w, c, src_coff=s_coff, dst_coff=d_coff)
    _sync()
    ref, bound = bilinear_reference(x, h, w)
    got = out[:, 1:-1, 1:-1, d_coff:d_coff + c].permute(0, 3, 1, 2)
    _check(f"upsample_bilinear {dtype} {hs}x{ws}->{h}x{w} c={c}", got, ref, _round16(bound, ref, dtype))
    assert bool((out[_outside(out, n, h, w, d_coff, c)] == SENT).all()), "written outside the window"


PLANE_CASES = [
    (1, 180, 320, 720, 1280),  # x4, the S2M output at 720p
    (2, 7, 5, 10, 13),
    (1, 13, 9, 5, 4),
    (1, 1, 1, 6, 8),
    (1, 6, 8, 1, 1),
]


@pytest.mark.parametrize("sig", [False, True])
@pytest.mark.parametrize("case", range(len(PLANE_CASES)))
def test_upsample_to_plane(dev, sig, case):
    """One channel (5 of 7; NaN in the others and the border) of an fp32 HALO map -> NCHW planes.  A quarter of the
    logits sit at +-30, where the sigmoid saturates.  One element past the planes must keep the sentinel."""
    n, hs, ws, H, W = PLANE_CASES[case]
    g = torch.Generator().manual_seed(100 + case)
    x = torch.randn(n, 1, hs, ws, generator=g) * 3
    pick = torch.randint(0, 8, x.shape, generator=g)
    x = torch.where(pick == 0, torch.full_like(x, 30.0), torch.where(pick == 1, torch.full_like(x, -30.0), x)).to(dev)
    halo = _halo(x, 7, 5, fill=NAN)
    buf = torch.full((n * H * W + 1,), SENT, device=dev)
    got = ops.halo_upsample_to_plane(halo, n, hs, ws, H, W, coff=5, sigmoid=sig, out=buf[:-1].view(n, 1, H, W))
    _sync()
    assert float(buf[-1]) == SENT
    ref, bound = bilinear_reference(x, H, W)
    if sig:
        p = torch.sigmoid(ref)
        ref, bound = p, p * (1 - p) * bound + p * (2 * U + 4 * U * (1 - p))
    _check(f"upsample_to_plane {hs}x{ws}->{H}x{W} sigmoid={sig}", got, ref, bound)


@pytest.mark.parametrize("act", ["fp16", "tf32"])
def test_conv_into_channel_window_with_ragged_cout(dev, act):
    """classifier.project: 1x1 256 -> 48 (+ReLU) written into channels [0, 48) of the 320-channel head
    buffer; channels 48.. must stay untouched."""
    dt = DT[act]
    g = torch.Generator().manual_seed(5)
    n, h, w = 2, 24, 32
    x = torch.randn((n, 256, h, w), generator=g)
    wt = torch.randn((48, 256, 1, 1), generator=g) / 16
    b = torch.randn((48,), generator=g)
    pc = ops.pack_conv(wt, b, device=dev, dtype=dt)
    assert (pc.cout, pc.cout_pad) == (48, 64)
    out = torch.full((n, h + 2, w + 2, 320), 7.0, device=dev, dtype=dt)
    ops.conv_gemm(to_halo(x.to(dev), dtype=dt), pc, n, h, w, out, relu=True)
    _sync()
    xr = x.half().float() if act == "fp16" else x
    want = torch.nn.functional.conv2d(xr.double(), pc.weight[0, :48, :256].double().cpu().view(48, 256, 1, 1), b.double()).relu()
    got = out[:, 1:-1, 1:-1, :48].permute(0, 3, 1, 2).double().cpu()
    assert float((got - want).abs().max()) <= 4e-3 * float(want.abs().max())
    assert bool((out[..., 48:] == 7).all()) and bool((out[:, 0] == 7).all())


# ------------------------------------------------------------------------------------------ network
@pytest.fixture(scope="module", params=["fp16", "tf32"])
def s2m_net(request, dev):
    import mivos_b200
    from oracle import weights
    net = mivos_b200.S2MNetwork(act_dtype=DT[request.param])
    net.load_state_dict(weights.make_s2m_state_dict(), strict=True)
    return net.to(dev)


def test_s2m_network_matches_reference_golden(golden, s2m_net, dev):
    g = golden("s2m_net.npz")
    x = torch.from_numpy(g["x"]).to(dev)
    before = int(_lib.load().mivos_launch_count())
    logits = s2m_net(x)
    _sync()
    assert int(_lib.load().mivos_launch_count()) - before > 60  # the whole pass ran through the C ABI
    ref = torch.from_numpy(g["logits"])
    assert logits.shape == ref.shape and logits.dtype == torch.float32
    eng = s2m_net.engine()
    H, W = x.shape[-2:]
    low = eng.ws.halo("low", 1, H // 4, W // 4, 256)[:, 1:-1, 1:-1].permute(0, 3, 1, 2).float().cpu()
    proj = eng.ws.halo("aspp_proj", 1, H // 16, W // 16, 256)[:, 1:-1, 1:-1].permute(0, 3, 1, 2).float().cpu()
    for name, got, want, tol in (("low_level", low, torch.from_numpy(g["low_level"]).float(), 1e-2),
                                 ("aspp", proj, torch.from_numpy(g["aspp"]), 1e-2),
                                 ("logits", logits.cpu(), ref, 2e-2)):
        err = float((got - want).abs().max()) / float(want.abs().max())
        print(f"s2m {name}: rel err {err:.2e}")
        assert err <= tol, (name, err)
    prob = s2m_net.forward_sigmoid(x).cpu()
    _sync()
    assert float((prob - torch.sigmoid(ref)).abs().max()) <= 3e-2
    assert float(((prob > 0.5) != (ref > 0)).float().mean()) <= 1e-2
    # a batch is the per-image result (objects of one interaction are batched); tile widths / split-K
    # factors depend on the row count, so the accumulation order — not the value — may differ
    p2 = s2m_net.forward_sigmoid(torch.cat([x.flip(-1), x], 0))
    _sync()
    assert float((p2[1:2].cpu() - prob).abs().max()) <= 5e-3


def test_s2m_controller_matches_reference_golden(golden, s2m_net, dev):
    from interact.s2m_controller import S2MController
    g = golden("s2m_controller.npz")
    ctrl = S2MController(s2m_net, int(g["k"]), ignore_class=255, device=dev)
    m = ctrl.interact(torch.from_numpy(g["image"]), torch.from_numpy(g["prev"]), g["scr"])
    _sync()
    ref = torch.from_numpy(g["mask"])
    assert m.shape == ref.shape and m.is_cuda
    assert float((m.cpu() - ref).abs().max()) <= 3e-2
    assert float(((m.cpu() > 0.5) != (ref > 0.5)).float().mean()) <= 1e-2


def test_s2m_feeds_the_propagation_path(nets, s2m_net, dev):
    """davis_processor.py:52-82: S2M probabilities -> aggregate_wbg(hard) -> InferenceCore.interact."""
    import mivos_b200
    from mivos_b200 import synth
    images, _ = synth.synthetic_clip(4, 96, 128, 2, seed=5)
    core = mivos_b200.InferenceCore(nets[20], None, images, 2, mem_freq=2, device=str(dev))
    scr = np.full((96, 128), 255, dtype=np.uint8)
    scr[30:33, 20:70] = 1
    scr[60:63, 50:110] = 2
    ctrl = mivos_b200.S2MController(s2m_net, 2, ignore_class=255, device=dev)
    prob = ctrl.interact(core.get_image_buffered(1), core.masks[1], scr)
    mask = mivos_b200.aggregate_wbg(prob, keep_bg=True, hard=True)
    out = core.interact(mask, 1)
    _sync()
    assert out.shape == (4, 96, 128) and out.dtype == np.uint8 and int(out.max()) <= 2
