"""CPU: the conv census checker (tests/conv_census.py) has teeth.

The float64 restatement of the ABI equals F.conv2d of the same rounded operands on small real layer forms; the checks
accept the fp32 emulation of tests/abi_emulator.py (another summation order) and reject each emulated kernel bug:
a dropped k-block, a dropped split-K partial, a tap reading across an image boundary, a misplaced residual, a skipped
bias tile, writes outside the window, and a truncated instead of rounded TF32 output."""
import dataclasses

import pytest
import torch
import torch.nn.functional as F

import abi_emulator as E
import conv_census as CC
from mivos_b200 import ops

H16, F32 = torch.float16, torch.float32
DTYPES = {"tf32": F32, "fp16": H16}


def _rounded_weight(wt, dtype):
    """The packed weight values (no BatchNorm) as an fp64 conv kernel."""
    return wt.half().double() if dtype == H16 else ops.round_tf32(wt.float()).double()


def _halo(x, cstride, coff=0, dtype=F32, fill=0.0):
    n, c, h, w = x.shape
    hb = torch.full((n, h + 2, w + 2, cstride), fill, dtype=dtype)
    hb[:, 1:-1, 1:-1, coff:coff + c] = x.permute(0, 2, 3, 1).to(dtype)
    if fill:
        hb[:, 0], hb[:, -1], hb[:, :, 0], hb[:, :, -1] = 0, 0, 0, 0
    return hb


def _rand(g, *shape, scale=1.0):
    return torch.randn(shape, generator=g) * scale


def _reference_nchw(L, ho, wo):
    y = CC.reference(L, CC.interior_rows(L.n, L.h, L.w, "cpu"))
    return y.reshape(L.n, ho, wo, -1).permute(0, 3, 1, 2)


def _close(y, ref):
    rel = float((y - ref).abs().max()) / float(ref.abs().max())
    assert rel <= 1e-12, rel


# ------------------------------------------------------------------ the reference is right
@pytest.mark.parametrize("act", list(DTYPES))
def test_reference_3x3_halo_three_images(act):
    dt = DTYPES[act]
    g = torch.Generator().manual_seed(1)
    n, h, w, cin, cout = 3, 7, 11, 40, 72
    x, wt, b = _rand(g, n, cin, h, w), _rand(g, cout, cin, 3, 3, scale=0.1), _rand(g, cout)
    pc = ops.pack_conv(wt, b, device="cpu", dtype=dt)
    xh = _halo(x, pc.cin_pad, dtype=dt)
    L = CC.snapshot(xh, pc, n, h, w, torch.zeros((n, h + 2, w + 2, pc.cout_pad)), relu=True)
    CC.check_premises(L)
    ref = F.conv2d(CC.operand64(x.to(dt)), _rounded_weight(wt, dt), b.double(), padding=1).relu()
    _close(_reference_nchw(L, h, w), ref)


@pytest.mark.parametrize("act", list(DTYPES))
def test_reference_stride2_gather_one_tap(act):
    dt = DTYPES[act]
    g = torch.Generator().manual_seed(2)
    n, h, w, cin, cout = 2, 10, 14, 32, 64
    x, wt, b = _rand(g, n, cin, h, w), _rand(g, cout, cin, 3, 3, scale=0.1), _rand(g, cout)
    pc = ops.pack_conv(wt, b, stride=2, im2col=True, device="cpu", dtype=dt)
    ho, wo = h // 2, w // 2
    mat = torch.zeros((n * (ho + 2) * (wo + 2), pc.cin_pad), dtype=dt)
    E.gather_s2(_halo(x, cin, dtype=dt), n, h, w, cin, 3, mat)
    L = CC.snapshot(mat, pc, n, ho, wo, torch.zeros((n, ho + 2, wo + 2, pc.cout_pad)))
    CC.check_premises(L)
    ref = F.conv2d(CC.operand64(x.to(dt)), _rounded_weight(wt, dt), b.double(), stride=2, padding=1)
    _close(_reference_nchw(L, ho, wo), ref)


@pytest.mark.parametrize("act", list(DTYPES))
def test_reference_s2d_stem_four_taps(act):
    """n = 2: tap dy = -2 of image 1's first lines reads image 0's bottom border (zero), not image 0's last line."""
    dt = DTYPES[act]
    g = torch.Generator().manual_seed(3)
    n, H, W, cin, cout = 2, 12, 20, 5, 64
    x, wt, b = _rand(g, n, cin, H, W), _rand(g, cout, cin, 7, 7, scale=0.05), _rand(g, cout)
    pc = ops.pack_conv(wt, b, stride=2, stem_s2d=True, device="cpu", dtype=dt)
    assert pc.taps == 4 and pc.cin_pad == (96 if dt == F32 else 128)
    ho, wo = H // 2, W // 2
    mat = torch.zeros((n * (ho + 2) * (wo + 2), pc.cin_pad), dtype=dt)
    E.stem_gather(x.to(dt).float(), None, mat, s2d=True)
    L = CC.snapshot(mat, pc, n, ho, wo, torch.zeros((n, ho + 2, wo + 2, pc.cout_pad)))
    CC.check_premises(L)
    ref = F.conv2d(CC.operand64(x.to(dt)), _rounded_weight(wt, dt), b.double(), stride=2, padding=3)
    _close(_reference_nchw(L, ho, wo), ref)


@pytest.mark.parametrize("act", list(DTYPES))
def test_reference_dilated_one_tap(act):
    dt = DTYPES[act]
    g = torch.Generator().manual_seed(4)
    n, h, w, cin, cout, d = 2, 9, 13, 32, 32, 3
    x, wt, b = _rand(g, n, cin, h, w), _rand(g, cout, cin, 3, 3, scale=0.1), _rand(g, cout)
    pc = ops.pack_conv(wt, b, im2col=True, device="cpu", dtype=dt)
    mat = torch.zeros((n * (h + 2) * (w + 2), pc.cin_pad), dtype=dt)
    E.gather_dilated(_halo(x, cin, dtype=dt), n, h, w, cin, d, mat)
    L = CC.snapshot(mat, pc, n, h, w, torch.zeros((n, h + 2, w + 2, pc.cout_pad)))
    CC.check_premises(L)
    ref = F.conv2d(CC.operand64(x.to(dt)), _rounded_weight(wt, dt), b.double(), padding=d, dilation=d)
    _close(_reference_nchw(L, h, w), ref)


@pytest.mark.parametrize("act", list(DTYPES))
def test_reference_channel_window_with_residual_window(act):
    dt = DTYPES[act]
    g = torch.Generator().manual_seed(5)
    n, h, w, cin, cout = 2, 6, 9, 64, 100
    x, wt, b, r = _rand(g, n, cin, h, w), _rand(g, cout, cin, 3, 3, scale=0.1), _rand(g, cout), _rand(g, n, cout, h, w)
    pc = ops.pack_conv(wt, b, device="cpu", dtype=dt)
    xh = _halo(x, 192, coff=64, dtype=dt, fill=7.0)  # channels outside [64, 128) are not the operand
    rh = _halo(r, 256, coff=96, dtype=dt, fill=5.0)
    out = torch.zeros((n, h + 2, w + 2, 320), dtype=dt)
    L = CC.snapshot(xh, pc, n, h, w, out, in_coff=64, out_coff=192, residual=rh, res_coff=96, relu=True)
    CC.check_premises(L)
    ref = (F.conv2d(CC.operand64(x.to(dt)), _rounded_weight(wt, dt), b.double(), padding=1) + r.to(dt).double()).relu()
    _close(_reference_nchw(L, h, w), ref)


# ------------------------------------------------------------------ emulated kernels and their mutations
def _emulated(x, pc, n, h, w, out, *, mutate=None, **kw):
    """abi_emulator.conv_gemm (fp32, its own summation order) on the operand the tensor core sees (fp32 truncated to
    TF32), plus the round_tf32 output rounding the emulator leaves out; `mutate(stage, value)` injects a bug."""
    x, pc, kw = (mutate("args", (x, pc, kw)) if mutate else (x, pc, kw))
    if x.dtype == F32:
        x = (x.contiguous().view(torch.int32) & ~CC.TF32_LOW).view(F32)
    E.conv_gemm(x, pc, n, h, w, out, **kw)
    win = CC.window(out, n, h, w, kw.get("out_coff", 0), pc.cout)
    if kw.get("round_tf32") and out.dtype == F32:
        win.copy_(mutate("round", win.clone()) if mutate else ops.round_tf32(win.clone()))
    if kw.get("out_relu") is not None:
        CC.window(kw["out_relu"], n, h, w, kw.get("out_relu_coff", 0), pc.cout).copy_(win.clamp_min(0))
    if mutate:
        mutate("out", out)
    return out


def _case(act, *, taps=9, n=3, h=7, w=11, cin=128, cout=100, res=True, dual=True, rnd=False, seed=9):
    """A layer with its operand (TF32-exact fp32 or fp16, so that the emulator multiplies what the kernel would),
    a residual window, a ReLU copy and an output window between neighbours filled with a sentinel."""
    dt = DTYPES[act]
    g = torch.Generator().manual_seed(seed)
    x = _rand(g, n, cin, h, w)
    x = x.half() if dt == H16 else ops.round_tf32(x)
    wt = _rand(g, cout, cin, 3 if taps == 9 else 1, 3 if taps == 9 else 1, scale=0.1)
    pc = ops.pack_conv(wt, _rand(g, cout), device="cpu", dtype=dt)
    kw = dict(out_coff=64, relu=not dual, round_tf32=rnd)
    if res:
        kw.update(residual=_halo(_rand(g, n, cout, h, w), 256, coff=32, dtype=dt, fill=3.0), res_coff=32)
    if dual:
        kw.update(out_relu=torch.full((n, h + 2, w + 2, 192), -7.0, dtype=dt), out_relu_coff=40)
    out = torch.full((n, h + 2, w + 2, 256), -7.0, dtype=dt)
    return _halo(x.float(), pc.cin_pad, dtype=dt), pc, n, h, w, out, kw


def _run(kernel, case, max_macs=CC.SAMPLE_MACS):
    x, pc, n, h, w, out, kw = case
    L = CC.snapshot(x, pc, n, h, w, out, layer="case", **kw)
    kernel(x, pc, n, h, w, out, **kw)
    return CC.check_launch(L, out, kw.get("out_relu"), max_macs=max_macs)


@pytest.mark.parametrize("max_macs", [CC.SAMPLE_MACS, 0], ids=["all_rows", "sampled"])
@pytest.mark.parametrize("act,rnd", [("tf32", False), ("tf32", True), ("fp16", False)])
def test_check_accepts_the_emulator(act, rnd, max_macs):
    rec = _run(_emulated, _case(act, rnd=rnd), max_macs)
    assert 0.0 < rec["ratio"] <= 1.0 and rec["sampled"] == (max_macs == 0)
    rec = _run(_emulated, _case(act, taps=1, res=False, dual=False, rnd=rnd), max_macs)
    assert rec["ratio"] <= 1.0


def _drop_last_kblock(stage, v):
    if stage == "args":
        x, pc, kw = v
        kq = 64 if pc.weight.dtype == H16 else 32
        wt = pc.weight.clone()
        wt[-1, :, pc.cin_pad - kq:] = 0
        return x, dataclasses.replace(pc, weight=wt), kw
    return v


def _drop_split(stage, v, S=3, s=1):
    """Split-K over S parts of the flattened (tap, k-block) axis; partial s never reaches the sum."""
    if stage == "args":
        x, pc, kw = v
        kq = 64 if pc.weight.dtype == H16 else 32
        nb = pc.taps * pc.cin_pad // kq
        lo, hi = s * nb // S * kq, (s + 1) * nb // S * kq
        wt = pc.weight.clone().permute(1, 0, 2).reshape(pc.cout_pad, -1)
        wt[:, lo:hi] = 0
        return x, dataclasses.replace(pc, weight=wt.reshape(pc.cout_pad, pc.taps, pc.cin_pad).permute(1, 0, 2).contiguous()), kw
    return v


def _prev_image_row(stage, v):
    """Tap dy = -1 of an image's first line reads the previous image's last interior line instead of its border."""
    if stage == "args":
        x, pc, kw = v
        x = x.clone()
        x[1:, 0] = x[:-1, -2]
        return x, pc, kw
    return v


def _residual_row_off(stage, v):
    if stage == "args":
        x, pc, kw = v
        r = kw["residual"]
        flat = r.reshape(-1, r.shape[-1])
        return x, pc, dict(kw, residual=torch.cat([flat[1:], flat[-1:]]).view(r.shape))
    return v


def _residual_chan_off(stage, v):
    if stage == "args":
        x, pc, kw = v
        return x, pc, dict(kw, res_coff=kw["res_coff"] + 4)
    return v


def _bias_last_tile(stage, v):
    if stage == "args":
        x, pc, kw = v
        b = pc.bias.clone()
        b[(pc.cout - 1) // 32 * 32:] = 0
        return x, dataclasses.replace(pc, bias=b), kw
    return v


def _border_write(stage, v):
    if stage == "out":
        v[1, 0, 3, 70] = 0.5
    return v


def _past_cout_write(stage, v):
    if stage == "out":
        v[0, 2, 5, 64 + 100] = 0.5  # first channel of the neighbouring window
    return v


def _truncate_tf32(stage, v):
    if stage == "round":
        return (v.contiguous().view(torch.int32) & ~CC.TF32_LOW).view(F32)
    return v


MUTATIONS = {
    "last_kblock_of_last_tap_dropped": (_drop_last_kblock, {}),
    "split_partial_dropped_S3": (_drop_split, {}),
    "dy_minus1_reads_previous_image": (_prev_image_row, {}),
    "residual_one_row_off": (_residual_row_off, {}),
    "residual_4_channels_off": (_residual_chan_off, {}),
    "bias_skipped_on_last_32_tile": (_bias_last_tile, {}),
    "border_element_written": (_border_write, {}),
    "element_past_cout_written": (_past_cout_write, {}),
    "round_tf32_truncated": (_truncate_tf32, dict(rnd=True, dual=False)),
}


@pytest.mark.parametrize("max_macs", [CC.SAMPLE_MACS, 0], ids=["all_rows", "sampled"])
@pytest.mark.parametrize("mutation,act", [(m, a) for m in MUTATIONS for a in DTYPES
                                          if not (m == "round_tf32_truncated" and a == "fp16")])  # fp32 outputs only
def test_check_rejects_mutation(mutation, act, max_macs):
    fn, extra = MUTATIONS[mutation]
    case = _case(act, **extra)
    _run(_emulated, case, max_macs)  # the unmutated kernel passes on the same case
    with pytest.raises(AssertionError):
        _run(lambda *a, **k: _emulated(*a, mutate=fn, **k), _case(act, **extra), max_macs)


@pytest.mark.parametrize("act", list(DTYPES))
def test_check_rejects_a_write_into_the_next_chunk(act):
    """`out` is the chunk view lg[k0:k0 + n] of a logits map of more objects: a kernel that writes one element into
    the next chunk's first map writes inside the allocation but outside the view, and must fail."""
    x, pc, n, h, w, out, kw = _case(act, res=False, dual=False)
    parent = torch.full((2 * n + 2, h + 2, w + 2, out.shape[-1]), -7.0, dtype=out.dtype)
    chunk = parent[2:2 + n]
    rec = _run(_emulated, (x, pc, n, h, w, chunk, kw))
    assert rec["ratio"] <= 1.0 and rec["alloc_maps"] == 2 * n + 2

    def spill(stage, v):
        if stage == "out":
            parent[2 + n, 3, 4, 64] = 0.5  # interior element of the window's channels, one map past the view
        return v
    parent.fill_(-7.0)
    with pytest.raises(AssertionError, match="outside the view"):
        _run(lambda *a, **k: _emulated(*a, mutate=spill, **k), (x, pc, n, h, w, chunk, kw))


def test_premise_checks_reject_dirty_operands():
    x, pc, n, h, w, out, kw = _case("tf32")
    x[0, 0, 4, 3] = 1.0  # a HALO border element of the operand
    with pytest.raises(AssertionError, match="border"):
        CC.check_premises(CC.snapshot(x, pc, n, h, w, out, **kw))
    x, pc, n, h, w, out, kw = _case("tf32")
    x[1, 3, 4, 0] = float("nan")
    with pytest.raises(AssertionError, match="finite"):
        CC.check_premises(CC.snapshot(x, pc, n, h, w, out, **kw))
    x, pc, n, h, w, out, kw = _case("tf32", cin=100)
    pc.weight[2, 5, 110] = 1.0  # past the real K of a tap
    with pytest.raises(AssertionError, match="past K"):
        CC.check_premises(CC.snapshot(x, pc, n, h, w, out, **kw))


def test_sample_rows_cover_tile_edges_and_image_lines():
    n, h, w = 3, 40, 70
    rows = CC.sample_rows(n, h, w, "cpu", seed=1)
    total = n * (h + 2) * (w + 2)
    assert bool(CC.interior_mask(rows, n, h, w).all()) and rows.unique().numel() == rows.numel()
    got = set(rows.tolist())
    inner = set(CC.interior_rows(n, h, w, "cpu").tolist())
    last = (total + CC.BM - 1) // CC.BM - 1
    for t in (0, 1, last - 1, last):
        assert set(range(t * CC.BM, min((t + 1) * CC.BM, total))) & inner <= got
    for m0 in range(0, total, CC.BM):
        assert {m0, m0 + 63, m0 + 64, m0 + 127} & inner <= got
    P = (h + 2) * (w + 2)
    for i in range(n):
        assert {i * P + (w + 2) + c for c in range(1, w + 1)} <= got and {i * P + h * (w + 2) + c for c in range(1, w + 1)} <= got


def test_census_records_a_real_engine(monkeypatch):
    """FusionEngine on the emulator, through Census.record: every launch labelled with its layer, checked, and a
    repeated launch counted but not checked again."""
    from mivos_b200 import engine as eng
    from oracle import weights as Wt
    E.install(monkeypatch, ops)
    monkeypatch.setattr(ops, "conv_gemm", _emulated)
    fe = eng.FusionEngine(Wt.make_fusion_state_dict(4321), "cpu")
    census = CC.Census()
    census.label(fe.pc, "fusion.")
    g = torch.Generator().manual_seed(6)
    H, W = 24, 40
    planes = [torch.rand((1, c, H, W), generator=g) for c in (3, 1, 1, 2)]
    with census.record("fusion"):
        for _ in range(2):
            fe.forward_logit_halo(*planes, 0.5, 0.25)
    assert census.seen["fusion"] == 12 and census.checked["fusion"] == 6
    assert [r["layer"] for r in census.records] == ["fusion." + k for k in ("conv1.0", "conv2.0", "conv2.2", "conv3.0",
                                                                            "conv3.2", "final_conv")]
    assert all(r["ratio"] <= 1.0 for r in census.records)
    assert ops.conv_gemm is _emulated
    print("\n" + census.table())
