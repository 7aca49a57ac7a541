"""GPU: the object-group forms of the operators whose operands differ per lock-step clip (mivos_*_groups).  Groups
of ragged sizes (1, 5, 2, 16, 3 objects, and one group alone) must give, bit for bit, what the existing operator gives
run once per group on that group's slice — the existing forms are held to float64 references in their own tests —
and the uniform table first = [0, K, 2K, ...] must give the bits of the existing per-set / groups / skip_n / src_n
form."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402

SIZES = [1, 5, 2, 16, 3]
H16, W16 = 14, 20        # hw = 280: one bank frame holds more slots than the widest top-k tested
HW = H16 * W16
CAP_FRAMES = 4


def _first(sizes, dev):
    f = [0]
    for k in sizes:
        f.append(f[-1] + k)
    return torch.tensor(f, dtype=torch.int32, device=dev), f


@pytest.fixture(autouse=True)
def _clean_kernel_errors():
    yield
    torch.cuda.synchronize()
    _lib.poll_kernel_error()


# ---- memory reads ------------------------------------------------------------------------------------------------

READS = [("topk", 1), ("topk", 20), ("topk", 64), ("wide", 100), ("dense", None)]


def _counts(kind, k, groups):
    """Live slots per group: the whole bank, the top-k bound itself, and partial frames."""
    bound = 1 if k is None else k
    base = [CAP_FRAMES * HW, bound, 2 * HW, HW, 3 * HW - 7]
    return [base[g % len(base)] for g in range(groups)]


def _bank(seed, dev, sizes, counts):
    g = torch.Generator().manual_seed(seed)
    K, cap = sum(sizes), CAP_FRAMES * HW
    bk = torch.randn((K, cap, 128), generator=g)
    bv = torch.randn((K, cap, 512), generator=g)
    o = 0
    for n, c in zip(sizes, counts):  # slots past a group's count hold NaN: they must take no part
        bk[o:o + n, c:] = float("nan")
        bv[o:o + n, c:] = float("nan")
        o += n
    qk = torch.randn((len(sizes), HW, 128), generator=g)
    return bk.to(dev), bv.to(dev), qk.to(dev)


def _ws(kind, k, K, dev):
    cap = CAP_FRAMES * HW
    n = (ops.memory_read_workspace_bytes(K, cap, HW, k) if kind == "topk" else
         ops.memory_read_wide_workspace_bytes(K, cap, HW, k) if kind == "wide" else
         ops.memory_read_dense_workspace_bytes(K, cap, HW))
    return torch.empty(n, dtype=torch.uint8, device=dev)


def _grouped(kind, k, bk, bv, qk, counts, first, out, ws):
    slots = bk.shape[1]
    if kind == "topk":
        ops.memory_read_groups(bk, bv, slots, qk, k, out, counts, first, workspace=ws)
    elif kind == "wide":
        ops.memory_read_wide_groups(bk, bv, slots, qk, k, out, counts, first, workspace=ws)
    else:
        ops.memory_read_dense_groups(bk, bv, slots, qk, out, counts, first, workspace=ws)
    return out


def _scalar(kind, k, bk, bv, slots, qk, out):
    if kind == "topk":
        ops.memory_read(bk, bv, slots, qk, k, out)
    elif kind == "wide":
        ops.memory_read_wide(bk, bv, slots, qk, k, out)
    else:
        ops.memory_read_dense(bk, bv, slots, qk, out)
    return out


@pytest.mark.parametrize("sizes", [SIZES, [16]], ids=["ragged", "one-group"])
@pytest.mark.parametrize("kind,k", READS)
def test_grouped_read_equals_one_read_per_group(dev, kind, k, sizes):
    counts = _counts(kind, k, len(sizes))
    bk, bv, qk = _bank(21, dev, sizes, counts)
    first, f = _first(sizes, dev)
    K = f[-1]
    out = torch.full((K, HW, 512), 7.0, device=dev)
    _grouped(kind, k, bk, bv, qk, torch.tensor(counts, dtype=torch.int32, device=dev), first, out, _ws(kind, k, K, dev))
    ref = torch.empty_like(out)
    for g, c in enumerate(counts):
        o = slice(f[g], f[g + 1])
        _scalar(kind, k, bk[o].contiguous(), bv[o].contiguous(), c, qk[g].contiguous(), ref[o])
    torch.cuda.synchronize()
    assert not torch.isnan(out).any()
    assert torch.equal(out, ref)


@pytest.mark.parametrize("kind,k", READS)
def test_grouped_read_with_a_uniform_table_gives_the_per_set_bits(dev, kind, k):
    sets, per = 4, 3
    counts = _counts(kind, k, sets)
    bk, bv, qk = _bank(22, dev, [per] * sets, counts)
    first, _ = _first([per] * sets, dev)
    cnt = torch.tensor(counts, dtype=torch.int32, device=dev)
    out = torch.empty((sets * per, HW, 512), device=dev)
    _grouped(kind, k, bk, bv, qk, cnt, first, out, _ws(kind, k, sets * per, dev))
    ref = torch.empty_like(out)
    ws = _ws(kind, k, sets * per, dev)
    if kind == "topk":
        ops.memory_read_sets(bk, bv, bk.shape[1], qk, k, ref, cnt, workspace=ws)
    elif kind == "wide":
        ops.memory_read_wide_sets(bk, bv, bk.shape[1], qk, k, ref, cnt, workspace=ws)
    else:
        ops.memory_read_dense_sets(bk, bv, bk.shape[1], qk, ref, cnt, workspace=ws)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


@pytest.mark.parametrize("kind,k", [("topk", 20), ("dense", None)])
def test_grouped_read_graph_replay_follows_table_and_counts(dev, kind, k):
    K = sum(SIZES)
    bk, bv, qk = _bank(23, dev, SIZES, [CAP_FRAMES * HW] * len(SIZES))
    first, _ = _first(SIZES, dev)
    counts = torch.tensor(_counts(kind, k, len(SIZES)), dtype=torch.int32, device=dev)
    out = torch.zeros((K, HW, 512), device=dev)
    ws = _ws(kind, k, K, dev)
    _grouped(kind, k, bk, bv, qk, counts, first, out, ws)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _grouped(kind, k, bk, bv, qk, counts, first, out, ws)
    for sizes in ([3, 2, 16, 5, 1], [5, 5, 5, 5, 7]):
        t, f = _first(sizes, dev)
        first.copy_(t)
        c = _counts(kind, k, len(sizes))[::-1]
        counts.copy_(torch.tensor(c, dtype=torch.int32))
        g.replay()
        ref = torch.empty_like(out)
        for gi, cg in enumerate(c):
            o = slice(f[gi], f[gi + 1])
            _scalar(kind, k, bk[o].contiguous(), bv[o].contiguous(), cg, qk[gi].contiguous(), ref[o])
        torch.cuda.synchronize()
        assert torch.equal(out, ref), sizes


# ---- bank write ---------------------------------------------------------------------------------------------------

def test_grouped_bank_write_lands_each_group_in_its_frame(dev):
    g = torch.Generator().manual_seed(5)
    h, w, cap_frames = 4, 6, 5
    hw = h * w
    first, f = _first(SIZES, dev)
    K = f[-1]
    halo = torch.zeros((K, h + 2, w + 2, 640))
    halo[:, 1:-1, 1:-1] = torch.randn((K, h, w, 640), generator=g)
    halo = halo.to(dev)
    bk = torch.full((K, cap_frames * hw, 128), -5.0, device=dev)
    bv = torch.full((K, cap_frames * hw, 512), -5.0, device=dev)
    frames = [3, 0, 4, 7, 1]  # group 3: outside [0, t_max = 4]: writes nothing
    ops.bank_write_groups(halo, K, h, w, 0, 128, bk, bv, cap_frames - 1,
                          torch.tensor(frames, dtype=torch.int32, device=dev), first)
    want_k = torch.full_like(bk, -5.0)
    want_v = torch.full_like(bv, -5.0)
    interior = halo[:, 1:-1, 1:-1].reshape(K, hw, 640)
    for gi, t in enumerate(frames):
        if t < cap_frames:
            o = slice(f[gi], f[gi + 1])
            want_k[o, t * hw:(t + 1) * hw] = interior[o, :, :128]
            want_v[o, t * hw:(t + 1) * hw] = interior[o, :, 128:]
    torch.cuda.synchronize()
    assert torch.equal(bk, want_k) and torch.equal(bv, want_v)


def test_grouped_bank_write_with_a_uniform_table_gives_the_per_set_bits(dev):
    g = torch.Generator().manual_seed(6)
    h, w, cap_frames, sets, per = 4, 6, 5, 4, 3
    halo = torch.randn((sets * per, h + 2, w + 2, 640), generator=g).to(dev)
    frames = torch.tensor([2, 0, 4, 1], dtype=torch.int32, device=dev)
    outs = []
    for grouped in (True, False):
        bk = torch.zeros((sets * per, cap_frames * h * w, 128), device=dev)
        bv = torch.zeros((sets * per, cap_frames * h * w, 512), device=dev)
        if grouped:
            ops.bank_write_groups(halo, sets * per, h, w, 0, 128, bk, bv, cap_frames - 1, frames,
                                  _first([per] * sets, dev)[0])
        else:
            ops.bank_write_sets(halo, sets * per, sets, h, w, 0, 128, bk, bv, cap_frames - 1, frames)
        outs.append((bk, bv))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


# ---- memorize stem --------------------------------------------------------------------------------------------------

def _packed_planes(sizes, H, W, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return torch.rand((sum(sizes) + len(sizes), 1, H, W), generator=g).to(dev)


@pytest.mark.parametrize("f16", [True, False])
def test_grouped_stem_gather_equals_one_gather_per_group(dev, f16):
    H, W = 48, 64
    dt = torch.float16 if f16 else torch.float32
    first, f = _first(SIZES, dev)
    K, G = f[-1], len(SIZES)
    frames = torch.randn((G, 3, H, W), generator=torch.Generator().manual_seed(7)).to(dev)
    planes = _packed_planes(SIZES, H, W, 8, dev)
    out = torch.full((K, H // 2 + 2, W // 2 + 2, 80), 3.0, dtype=dt, device=dev)
    ops.stem_gather_groups(frames, planes, K, first, out)
    ref = torch.empty_like(out)
    for gi in range(G):
        masks = planes[f[gi] + gi + 1:f[gi + 1] + gi + 1].contiguous()  # group gi's objects, after its background
        ops.stem_gather(frames[gi].contiguous(), masks, ref[f[gi]:f[gi + 1]], s2d=True)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


def test_grouped_stem_gather_with_a_uniform_table_gives_the_groups_bits(dev):
    H, W, G, per = 32, 48, 3, 4
    frames = torch.randn((G, 3, H, W), generator=torch.Generator().manual_seed(9)).to(dev)
    planes = _packed_planes([per] * G, H, W, 10, dev)
    out = torch.empty((G * per, H // 2 + 2, W // 2 + 2, 80), dtype=torch.float16, device=dev)
    ops.stem_gather_groups(frames, planes, G * per, _first([per] * G, dev)[0], out)
    ref = torch.empty_like(out)
    ops.stem_gather(frames, planes.view(G, per + 1, 1, H, W).narrow(1, 1, per), ref, s2d=True)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


# ---- skip broadcast and v16 copy -------------------------------------------------------------------------------------

@pytest.mark.parametrize("f16", [True, False])
def test_grouped_skip_broadcast_equals_one_call_per_group(dev, f16):
    h, w, c = 12, 16, 64
    dt = torch.float16 if f16 else torch.float32
    first, f = _first(SIZES, dev)
    K, G = f[-1], len(SIZES)
    g = torch.Generator().manual_seed(11)
    up = ops.halo_zeros(K, h // 2, w // 2, c, dev, dt)
    up[:, 1:-1, 1:-1] = torch.randn((K, h // 2, w // 2, c), generator=g).to(dev, dt)
    skip = ops.halo_zeros(G, h, w, c, dev, dt)
    skip[:, 1:-1, 1:-1] = torch.randn((G, h, w, c), generator=g).to(dev, dt)
    x, xr = ops.halo_zeros(K, h, w, c, dev, dt), ops.halo_zeros(K, h, w, c, dev, dt)
    ops.upsample2x_add_groups(x, up, K, h, w, skip, first, x_relu=xr)
    rx, rr = ops.halo_zeros(K, h, w, c, dev, dt), ops.halo_zeros(K, h, w, c, dev, dt)
    for gi in range(G):
        o = slice(f[gi], f[gi + 1])
        ops.upsample2x_add(rx[o], up[o], SIZES[gi], h, w, x_relu=rr[o], skip=skip[gi:gi + 1])
    # uniform table: the bits of skip_n
    xu = ops.halo_zeros(12, h, w, c, dev, dt)
    ops.upsample2x_add_groups(xu, up[:12], 12, h, w, skip[:3], _first([4, 4, 4], dev)[0])
    ru = ops.halo_zeros(12, h, w, c, dev, dt)
    ops.upsample2x_add(ru, up[:12], 12, h, w, skip=skip[:3])
    torch.cuda.synchronize()
    assert torch.equal(x, rx) and torch.equal(xr, rr)
    assert torch.equal(xu, ru)


@pytest.mark.parametrize("f16", [True, False])
def test_grouped_v16_copy_equals_one_copy_per_group(dev, f16):
    h, w = 7, 10
    dt = torch.float16 if f16 else torch.float32
    first, f = _first(SIZES, dev)
    K, G = f[-1], len(SIZES)
    src = torch.randn((G, h + 2, w + 2, 640), generator=torch.Generator().manual_seed(12)).to(dev, dt)
    dst = torch.full((K, h + 2, w + 2, 1024), 2.0, dtype=dt, device=dev)
    ops.halo_copy_groups(src, dst, K, h, w, 512, first, src_coff=128, dst_coff=512)
    ref = torch.full_like(dst, 2.0)
    for gi in range(G):
        o = slice(f[gi], f[gi + 1])
        ops.halo_copy(src[gi:gi + 1], ref[o], SIZES[gi], h, w, 512, src_coff=128, dst_coff=512)
    du = torch.full((12, h + 2, w + 2, 1024), 2.0, dtype=dt, device=dev)
    ops.halo_copy_groups(src[:3], du, 12, h, w, 512, _first([4, 4, 4], dev)[0], src_coff=128, dst_coff=512)
    ru = torch.full_like(du, 2.0)
    ops.halo_copy(src[:3], ru, 12, h, w, 512, src_coff=128, dst_coff=512)
    torch.cuda.synchronize()
    assert torch.equal(dst, ref)
    assert torch.equal(du, ru)


# ---- decoder tail and aggregation ----------------------------------------------------------------------------------

def _logits(K, h4, w4, seed, dev):
    g = torch.Generator().manual_seed(seed)
    lg = torch.zeros((K, h4 + 2, w4 + 2, 32))
    lg[:, 1:-1, 1:-1] = 3 * torch.randn((K, h4, w4, 32), generator=g)
    return lg.to(dev)


def _aggregate_f64(lg, h4, w4):
    """float64: bilinear x4 (align_corners=False), sigmoid, aggregate_wbg(keep_bg=True) of one group."""
    x = lg[:, 1:-1, 1:-1, 0].double().unsqueeze(1)
    p = torch.sigmoid(torch.nn.functional.interpolate(x, scale_factor=4, mode="bilinear", align_corners=False))
    bg = torch.prod(1 - p, dim=0, keepdim=True)
    v = torch.cat([bg, p], 0).clamp(1e-7, 1 - 1e-7)
    return torch.softmax(torch.log(v / (1 - v)), dim=0)


@pytest.mark.parametrize("sizes", [SIZES, [16]], ids=["ragged", "one-group"])
def test_grouped_aggregation_equals_one_call_per_group(dev, sizes):
    h4, w4 = 9, 13
    H, W = 4 * h4, 4 * w4
    first, f = _first(sizes, dev)
    K, G = f[-1], len(sizes)
    lg = _logits(K, h4, w4, 13, dev)
    raw = torch.full((K, 1, H, W), 5.0, device=dev)
    prob = torch.full((K + G, 1, H, W), 5.0, device=dev)
    ops.upsample4x_sigmoid_aggregate_groups(lg, K, h4, w4, first, raw_out=raw, prob_out=prob)
    rraw, rprob = torch.empty_like(raw), torch.empty_like(prob)
    for gi in range(G):
        ops.upsample4x_sigmoid_aggregate(lg[f[gi]:f[gi + 1]].contiguous(), sizes[gi], h4, w4,
                                         raw_out=rraw[f[gi]:f[gi + 1]], prob_out=rprob[f[gi] + gi:f[gi + 1] + gi + 1])
    torch.cuda.synchronize()
    assert torch.equal(raw, rraw) and torch.equal(prob, rprob)
    for gi in range(G):  # and the float64 reference, at the tolerance of the register kernel's own tests
        want = _aggregate_f64(lg[f[gi]:f[gi + 1]].cpu(), h4, w4)
        got = prob[f[gi] + gi:f[gi + 1] + gi + 1].double().cpu()
        assert (got - want).abs().max() <= 1e-4, gi


def test_grouped_aggregation_with_a_uniform_table_gives_the_groups_bits(dev):
    h4, w4, G, per = 8, 12, 3, 5
    lg = _logits(G * per, h4, w4, 14, dev)
    _, prob = ops.upsample4x_sigmoid_aggregate_groups(lg, G * per, h4, w4, _first([per] * G, dev)[0])
    _, ref = ops.upsample4x_sigmoid_aggregate(lg, per, h4, w4, groups=G)
    torch.cuda.synchronize()
    assert torch.equal(prob, ref.reshape(prob.shape))


# ---- the mixed-object session ---------------------------------------------------------------------------------------
# LockstepSession(mixed_objects=True) over clips of 1, 3, 2 and 5 objects, different length, mem_freq, first
# interaction, and a second interaction that fuses on some clips only, against each clip's own InferenceCore.  As in
# tests/test_gpu_ragged_lockstep.py: with the convolution plan pinned every clip gets the bits of its own run; with
# the automatic plan a batch of other map counts may pick other split-K orders, so the mean difference is held to
# 1e-3 (2e-3 with fusion) and the maximum to 0.1, with labels agreeing wherever the clip's own run decided them.

import numpy as np  # noqa: E402

import mivos_b200  # noqa: E402
from oracle import weights as Wt  # noqa: E402  (synthetic clips only)

# clip: (objects, length, mem_freq, first interaction, second interaction)
MIXED = [(1, 7, 2, 2, 6), (3, 9, 3, 4, 8), (2, 5, 1, 0, 0), (5, 6, 2, 5, 2)]


def _mixed_clips(h, w):
    return [Wt.synthetic_clip(t, h, w, k, seed=40 + i) for i, (k, t, *_r) in enumerate(MIXED)]


def _mixed_cores(net, fuse, clips):
    return [mivos_b200.InferenceCore(net, fuse, img, MIXED[i][0], mem_freq=MIXED[i][2], device="cuda:0")
            for i, (img, _m) in enumerate(clips)]


def _mixed(net, fuse, clips, rounds):
    solo, cores = _mixed_cores(net, fuse, clips), _mixed_cores(net, fuse, clips)
    sess = mivos_b200.LockstepSession(cores, mixed_objects=True)
    for r in range(rounds):
        idxs = [c[3 + r] for c in MIXED]
        masks = [(m if r == 0 else m.flip(-1)).contiguous() for _img, m in clips]
        for s, m, i in zip(solo, masks, idxs):
            s.interact(m, i)
        sess.interact(masks, idxs)
    return solo, cores


def _close(solo, cores, fused, tag):
    for i, (s, c) in enumerate(zip(solo, cores)):
        assert c.bank_trace == s.bank_trace, (tag, i)
        d = (c.prob - s.prob).abs()
        mx, mean = 1e-1, (2e-3 if fused else 1e-3)
        assert float(d.max()) <= mx and float(d.mean()) <= mean, (tag, i, float(d.max()), float(d.mean()))
        top2 = s.prob[:, :, 0].topk(2, dim=0).values
        decided = (top2[0] - top2[1]) > 2 * mx
        assert torch.equal(c.masks[:, 0][decided], s.masks[:, 0][decided]), (tag, i)


def test_mixed_session_gives_each_clips_own_bits_under_a_pinned_conv_plan(dev, nets, monkeypatch):
    clips = _mixed_clips(64, 96)
    monkeypatch.setenv("MIVOS_GRAPH", "0")  # eager: no graph captured under the pinned plan outlives this test
    lib = _lib.load()
    _lib.check(lib.mivos_conv_tile_override(32, 0), "mivos_conv_tile_override")
    try:
        solo, cores = _mixed(nets[20], nets["fuse"], clips, 2)
    finally:
        _lib.check(lib.mivos_conv_tile_override(0, 0), "mivos_conv_tile_override")
    for s, c in zip(solo, cores):
        assert c.bank_trace == s.bank_trace
        assert torch.equal(c.prob, s.prob) and torch.equal(c.masks, s.masks) and np.array_equal(c.np_masks, s.np_masks)


def test_mixed_session_equals_each_clips_own_run(dev, nets):
    clips = _mixed_clips(64, 96)
    solo, cores = _mixed(nets[20], nets["fuse"], clips, 2)
    _close(solo, cores, True, "auto plan")
    assert [len(c.interacted) for c in cores] == [2, 2, 1, 2]


def test_mixed_graph_replay_is_bit_identical_to_eager(dev, nets, monkeypatch):
    clips = _mixed_clips(64, 96)
    net = nets[20]
    res = []
    for graph in ("0", "1", "1"):  # eager, graph capture, cached graph replay
        monkeypatch.setenv("MIVOS_GRAPH", graph)
        if graph == "0":
            net.engine().__dict__.pop("_lock_steps", None)
        cores = _mixed_cores(net, nets["fuse"], clips)
        sess = mivos_b200.LockstepSession(cores, mixed_objects=True)
        sess.interact([m for _i, m in clips], [c[3] for c in MIXED])
        out = sess.interact([m.flip(-1).contiguous() for _i, m in clips], [c[4] for c in MIXED])
        res.append(([o.copy() for o in out], [c.prob.clone() for c in cores]))
        if graph == "0":
            net.engine().__dict__.pop("_lock_steps", None)  # the eager step must not serve the graph runs
    for out, probs in res[1:]:
        for i in range(len(MIXED)):
            assert torch.equal(probs[i], res[0][1][i]) and np.array_equal(out[i], res[0][0][i])


@pytest.fixture(scope="module", params=["tf32", "fp16"])
def wide_dense_nets(request, prop_sd, dev):
    out = {}
    for k in (None, 100):
        n = mivos_b200.PropagationNetwork(top_k=k, act_dtype=torch.float16 if request.param == "fp16" else torch.float32)
        n.load_state_dict(prop_sd, strict=True)
        out[k] = n.to(dev)
    return out


@pytest.mark.parametrize("top_k", [None, 100])
def test_mixed_session_on_dense_and_wide_networks(dev, wide_dense_nets, top_k):
    clips = _mixed_clips(160, 224)  # hw = 140: every read of the wide network has at least top_k live slots
    solo, cores = _mixed(wide_dense_nets[top_k], None, clips, 1)
    _close(solo, cores, False, f"top_k={top_k}")
