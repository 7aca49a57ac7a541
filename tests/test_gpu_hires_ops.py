"""GPU: the kernels that take frames above 720p — the streamed attention map and weights (csrc/attention.cu,
attention_stream_kernel) and the column-tiled 6-channel stem gather (csrc/halo_ops.cu, mivos_stem_gather_frames_tiled)
— against float64 statements of the same operations, with the rules of tests/test_gpu_ops_ragged.py: references from
the operands the kernel saw, outputs pre-filled with a sentinel that must survive outside the written region, inputs
the kernel must not read (rows past the keys, the pixels past the frames) holding NaN.

Streamed attention bound (DESIGN.md §6).  The logit s_ij is attention_kernel's fma chain (GAMMA S_ij, S_ij =
sum_c |mk_ic qk_jc| / sqrt(128)).  The kernel processes keys in tiles of SK = 128; after tile t it holds the running
maximum m_t (exact: a max of fp32 logits) and adds e_ij = expf(fl(s_ij - m_t)) to per-lane partial sums, which it
multiplies by c = fl(expf(fl(m_{t-1} - m_t))) whenever the maximum grows.  A rescale's error is common to every term
already accumulated, in the denominator and in both numerators alike, so it enters like a relative error of those
terms: the argument roundings telescope to u (max - m_t) <= u |L_ij - max_i L_ij|, and each rescale adds 2 ulp of
expf (4u).  Per term, relative:
    eps_ij = GAMMA (S_ij + max_i S_ij) + 2u |L_ij - Lmax_j| + 4u (1 + R_ij)
where R_ij bounds the rescales after key i's tile: tile k can raise the fp32 running maximum only if its largest logit
plus GAMMA max S can exceed the running maximum's lower bound (the largest earlier tile maximum minus its GAMMA max S).
Every lane partial takes one rounding per term and one per tile multiply: (5T + 6)u with T = ceil(hw / 128), including
the 5 levels of the warp tree.  The map is the W-weighted mean of the pooled masks (an error shared by all terms
cancels), as for the resident kernel; W's second pass uses the final maximum, so its exponentials carry the resident
kernel's eps, and only the denominator carries the streamed errors."""

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402
from op_references import SK, map_reference, stem_images, stem_matrix, weights_streamed_blocks  # noqa: E402
from test_gpu_ops_ragged import H16, NAN, SENT, _check, _check_stem, _stem_out  # noqa: E402


def _worst(what, ratios):
    r = max(ratios)
    print(f"{what}: max err/bound = {r:.3g}")
    return r


def _inputs(h16, w16, scale, seed, dev):
    g = torch.Generator().manual_seed(seed)
    hw = h16 * w16
    mk = torch.randn(hw, 128, generator=g) * scale
    qk = torch.randn(hw, 128, generator=g) * scale
    pos = torch.rand(1, 1, 16 * h16, 16 * w16, generator=g)
    neg = torch.rand(1, 1, 16 * h16, 16 * w16, generator=g)
    return mk.to(dev), qk.to(dev), pos.to(dev), neg.to(dev)


def _guarded(x, guard=4096):
    """x [n, ...] in a flat fp32 buffer followed by `guard` NaNs; returns (buffer, view)."""
    buf = torch.full((x.numel() + guard,), NAN, dtype=torch.float32, device=x.device)
    buf[:x.numel()] = x.reshape(-1)
    return buf, buf[:x.numel()].view(x.shape)


def _run_map(mk, qk, h16, w16, pos, neg):
    """mivos_attention_map_streamed on NaN-guarded operands into a sentinel-guarded output."""
    hw = h16 * w16
    (_, mkv), (_, qkv), (_, pv), (_, nv) = _guarded(mk), _guarded(qk), _guarded(pos), _guarded(neg)
    n = 2 * 256 * hw
    out = torch.full((n + 1024,), SENT, dtype=torch.float32, device=mk.device)
    scratch = torch.full((4 * hw + 64,), SENT, dtype=torch.float32, device=mk.device)
    _lib.check(_lib.lib().mivos_attention_map_streamed(ops._ptr(mkv), ops._ptr(qkv), h16, w16, ops._ptr(pv), ops._ptr(nv),
                                                        ops._ptr(out), ops._ptr(scratch), ops._stream()),
               "mivos_attention_map_streamed")
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    assert bool((out[n:] == SENT).all()) and bool((scratch[4 * hw:] == SENT).all()), "wrote past the output / scratch"
    return out[:n].view(1, 2, 16 * h16, 16 * w16)


@pytest.mark.parametrize("scale", [1.0, 4.0])  # x4: logits of std 16, peaked columns where the rescales matter
@pytest.mark.parametrize("h16,w16", [(1, 1), (7, 9), (64, 108), (31, 223), (68, 120), (90, 160), (135, 240)])
def test_attention_map_streamed(dev, h16, w16, scale):
    """hw = 1, 63 (one ragged tile, two CTAs of 32 queries, the second ragged), 6912 (the resident kernel's limit: both
    kernels must agree within their two bounds), 6913 (the first hw above it), 8160 (1080p), 14400 (1440p) and 32400
    (4K).  Each mistake a streamed softmax could make is evaluated on the same inputs and must exceed the bound: a
    softmax over the query axis and a missing rescale at both scales, a skipped last tile at x4 (where a key can
    dominate its column) — at unit scale it is reported, since 16 keys of 32400 at 4K stay within the bound."""
    hw = h16 * w16
    mk, qk, pos, neg = _inputs(h16, w16, scale, hw * 10 + int(scale), dev)
    out = _run_map(mk, qk, h16, w16, pos, neg)
    ref, bound, bound_r, bad = map_reference(mk, qk, h16, w16, pos, neg, mistakes=hw > SK)  # (one tile: none apply)
    _check(f"attention_map_streamed hw={hw} x{scale:g}", out, ref, bound)
    for name, alt in bad.items():
        r = float(((alt - ref).abs() / bound).max())
        print(f"  mistake {name} hw={hw} x{scale:g}: max |alt - ref| / bound = {r:.3g}")
        if name == "skip_last_tile" and scale == 1.0:
            continue  # reported only: at 4K the last tile holds 16 of 32400 keys (0.55 of the bound); x4 catches it
        assert r > 1.0, (name, r)
    if hw == 6912:
        res = ops.attention_map(mk, qk, h16, w16, pos, neg)
        torch.cuda.synchronize()
        _check(f"streamed vs resident hw={hw} x{scale:g}", out, res.double(), bound + bound_r)
        _check(f"attention_map (resident) hw={hw} x{scale:g}", res, ref, bound_r)


@pytest.mark.parametrize("scale", [1.0, 4.0])
@pytest.mark.parametrize("hw", [63, 6913, 8160])
def test_attention_weights_streamed(dev, hw, scale):
    """W [hw, hw] written row by row: against float64 in column blocks; a guard past the matrix keeps its sentinel."""
    g = torch.Generator().manual_seed(hw * 7 + int(scale))
    mk = (torch.randn(hw, 128, generator=g) * scale).to(dev)
    qk = (torch.randn(hw, 128, generator=g) * scale).to(dev)
    (_, mkv), (_, qkv) = _guarded(mk), _guarded(qk)
    out = torch.full((hw * hw + 1024,), SENT, dtype=torch.float32, device=dev)
    scratch = torch.full((4 * hw,), SENT, dtype=torch.float32, device=dev)
    _lib.check(_lib.lib().mivos_attention_weights_streamed(ops._ptr(mkv), ops._ptr(qkv), hw, ops._ptr(out),
                                                            ops._ptr(scratch), ops._stream()), "mivos_attention_weights_streamed")
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    assert bool((out[hw * hw:] == SENT).all()), "wrote past W"
    Wg = out[:hw * hw].view(hw, hw)
    ratios = []
    for j0, j1, W, Wb in weights_streamed_blocks(mk, qk):
        err = (Wg[:, j0:j1].double() - W).abs()
        ratios.append(float((err / Wb).max()))
    r = _worst(f"attention_weights_streamed hw={hw} x{scale:g}", ratios)
    assert r <= 1.0, r


def test_streamed_and_resident_limits_are_independent(dev):
    """The streamed kernels set their own opt-in limit once; calls in any order leave the resident kernel's limit as
    it was: resident at 6912, streamed, resident weights at 6904, streamed weights, resident map at 6912."""
    mk, qk, pos, neg = _inputs(64, 108, 1.0, 3, dev)
    a = ops.attention_map(mk, qk, 64, 108, pos, neg)
    s = ops.attention_map_streamed(mk, qk, 64, 108, pos, neg)
    ops.attention_weights(mk[:6904].contiguous(), qk[:6904].contiguous())
    ops.attention_weights_streamed(mk[:6904].contiguous(), qk[:6904].contiguous())
    b = ops.attention_map(mk, qk, 64, 108, pos, neg)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    assert torch.equal(a, b)
    s2 = ops.attention_map_streamed(mk, qk, 64, 108, pos, neg)
    assert torch.equal(s, s2)  # deterministic


# ------------------------------------------------------------------------------------------------ tiled stem
def _tiled(frames, kpad, dtype):
    """mivos_stem_gather_frames_tiled over NaN-guarded frames into a sentinel matrix with a guard row."""
    n, cin, H, W = frames.shape
    _, fv = _guarded(frames)
    buf, out = _stem_out(n, H, W, kpad, dtype, frames.device)
    _lib.check(_lib.lib().mivos_stem_gather_frames_tiled(ops._ptr(fv), n, H, W, ops._ptr(out), kpad, ops._f16(out),
                                                          ops._stream()), "mivos_stem_gather_frames_tiled")
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    return buf


@pytest.mark.parametrize("dtype", [torch.float32, H16])
def test_stem_gather_frames_tiled(dev, dtype):
    """Widths 1378 (first refused by the untiled stem in fp32; 689 output columns: 5 windows of 128 + 49), 1920
    (1080p, 7.5 windows) and 3840 (4K, 15 windows exactly): bit-exact against a float64 F.unfold, pad columns and border
    rows zero, guard row untouched.  A window offset off by one input pixel (windows after the first staged from
    x + 1) changes the reference at these inputs, so the bit-exact check catches it."""
    g = torch.Generator().manual_seed(1920)
    kpad = 320
    for n, H, W in ((2, 6, 1378), (1, 10, 1920), (2, 4, 3840)):
        frames = torch.randn(n, 6, H, W, generator=g).to(dev)
        img, bound = stem_images(frames)
        buf = _tiled(frames, kpad, dtype)
        _check_stem(f"stem_gather_frames_tiled {dtype} n={n} {H}x{W}", buf, img, bound, kpad, False, dtype)
        rounded = img.to(dtype).double()
        ref = stem_matrix(rounded, kpad, False).reshape(n, H // 2 + 2, W // 2 + 2, kpad)
        shifted = stem_matrix(F.pad(rounded, (0, 1))[..., 1:], kpad, False).reshape(n, H // 2 + 2, W // 2 + 2, kpad)
        off = ref.clone()
        off[:, :, 129:] = shifted[:, :, 129:]  # HALO column 129 = output column 128: the first of window 1
        diff = int((off != ref).sum())
        print(f"  mistake window offset off by one {W} px: {diff} differing elements")
        assert diff > 0


def test_stem_gather_frames_tiled_equals_untiled(dev):
    """At widths both entry points take (one window at 22 px, six at 1376 px) the matrices are identical, fp32."""
    g = torch.Generator().manual_seed(22)
    for n, H, W in ((2, 6, 22), (1, 6, 1376)):
        frames = torch.randn(n, 6, H, W, generator=g).to(dev)
        buf = _tiled(frames, 320, torch.float32)
        buf2, out2 = _stem_out(n, H, W, 320, torch.float32, dev)
        ops.stem_gather_frames(frames, out2)
        torch.cuda.synchronize()
        assert torch.equal(buf, buf2), (H, W)
        buf3, out3 = _stem_out(n, H, W, 320, torch.float32, dev)
        ops.stem_gather_frames_tiled(frames, out3)
        torch.cuda.synchronize()
        assert torch.equal(buf3, buf2), (H, W)
