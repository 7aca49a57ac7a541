"""GPU: the per-set forms of the memory reads (mivos_memory_read_sets / _dense_sets / _wide_sets) and of the bank write
(mivos_bank_write_sets).  A per-set read of S sets must give, bit for bit, what S scalar reads give — one per set, over
that set's objects, query and live slot count — with NaN in every slot past a set's count; with all counts equal it
must give the bits of the scalar read over all objects (q_div = objects per set, one device-side count)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402

H16, W16 = 14, 20        # hw = 280: one bank frame holds more slots than the widest top-k tested
HW = H16 * W16
SETS, PER = 4, 2         # 4 clips of 2 objects
CAP_FRAMES = 6
FRAMES = [1, 3, 6, 4]    # live bank frames per set: one frame to capacity in one call


def _bank(seed, dev, frames=FRAMES):
    g = torch.Generator().manual_seed(seed)
    K, cap = SETS * PER, CAP_FRAMES * HW
    bk = torch.randn((K, cap, 128), generator=g)
    bv = torch.randn((K, cap, 512), generator=g)
    for s, f in enumerate(frames):  # slots past a set's count hold NaN: they must take no part
        bk[s * PER:(s + 1) * PER, f * HW:] = float("nan")
        bv[s * PER:(s + 1) * PER, f * HW:] = float("nan")
    qk = torch.randn((SETS, HW, 128), generator=g)
    return bk.to(dev), bv.to(dev), qk.to(dev)


def _counts(frames, dev):
    return torch.tensor([f * HW for f in frames], dtype=torch.int32, device=dev)


READS = [("topk", 1), ("topk", 20), ("topk", 64), ("wide", 65), ("wide", 256), ("dense", None)]


def _ws(kind, k, dev):
    K, cap = SETS * PER, CAP_FRAMES * HW
    n = (ops.memory_read_workspace_bytes(K, cap, HW, k) if kind == "topk" else
         ops.memory_read_wide_workspace_bytes(K, cap, HW, k) if kind == "wide" else
         ops.memory_read_dense_workspace_bytes(K, cap, HW))
    return torch.empty(n, dtype=torch.uint8, device=dev)


def _per_set(kind, k, bk, bv, qk, counts, out, ws):
    slots = bk.shape[1]
    if kind == "topk":
        ops.memory_read_sets(bk, bv, slots, qk, k, out, counts, workspace=ws)
    elif kind == "wide":
        ops.memory_read_wide_sets(bk, bv, slots, qk, k, out, counts, workspace=ws)
    else:
        ops.memory_read_dense_sets(bk, bv, slots, qk, out, counts, workspace=ws)
    return out


def _scalar(kind, k, bk, bv, slots, qk, out, dyn_slots=None, q_div=0):
    if kind == "topk":
        ops.memory_read(bk, bv, slots, qk, k, out, dyn_slots=dyn_slots, q_div=q_div)
    elif kind == "wide":
        ops.memory_read_wide(bk, bv, slots, qk, k, out, dyn_slots=dyn_slots, q_div=q_div)
    else:
        ops.memory_read_dense(bk, bv, slots, qk, out, dyn_slots=dyn_slots, q_div=q_div)
    return out


def _per_set_reference(kind, k, bk, bv, qk, frames):
    """One scalar read per set: that set's objects, query and live slot count (eager host count)."""
    out = torch.empty((SETS * PER, HW, 512), device=bk.device)
    for s, f in enumerate(frames):
        o = slice(s * PER, (s + 1) * PER)
        _scalar(kind, k, bk[o].contiguous(), bv[o].contiguous(), f * HW, qk[s].contiguous(), out[o])
    return out


@pytest.mark.parametrize("kind,k", READS)
def test_per_set_read_equals_one_scalar_read_per_set(dev, kind, k):
    bk, bv, qk = _bank(11, dev)
    out = torch.full((SETS * PER, HW, 512), 7.0, device=dev)
    _per_set(kind, k, bk, bv, qk, _counts(FRAMES, dev), out, _ws(kind, k, dev))
    ref = _per_set_reference(kind, k, bk, bv, qk, FRAMES)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    assert not torch.isnan(out).any()
    assert torch.equal(out, ref)


@pytest.mark.parametrize("kind,k", READS)
def test_per_set_read_with_equal_counts_gives_the_scalar_bits(dev, kind, k):
    bk, bv, qk = _bank(12, dev, frames=[CAP_FRAMES] * SETS)
    for f in (1, 5):
        out = torch.empty((SETS * PER, HW, 512), device=dev)
        _per_set(kind, k, bk, bv, qk, _counts([f] * SETS, dev), out, _ws(kind, k, dev))
        ref = torch.empty_like(out)
        _scalar(kind, k, bk, bv, bk.shape[1], qk, ref, dyn_slots=torch.tensor([f * HW], dtype=torch.int32, device=dev),
                q_div=PER)
        torch.cuda.synchronize()
        _lib.poll_kernel_error()
        assert torch.equal(out, ref), f


@pytest.mark.parametrize("kind,k", [("topk", 20), ("wide", 65), ("dense", None)])
def test_per_set_read_graph_replay_follows_the_counts(dev, kind, k):
    bk, bv, qk = _bank(13, dev, frames=[CAP_FRAMES] * SETS)
    counts = _counts(FRAMES, dev)
    out = torch.zeros((SETS * PER, HW, 512), device=dev)
    ws = _ws(kind, k, dev)
    _per_set(kind, k, bk, bv, qk, counts, out, ws)  # first use configures the kernels
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _per_set(kind, k, bk, bv, qk, counts, out, ws)
    for frames in (FRAMES, [6, 1, 2, 5], [2, 2, 2, 2]):
        counts.copy_(_counts(frames, dev))
        g.replay()
        ref = _per_set_reference(kind, k, bk, bv, qk, frames)
        torch.cuda.synchronize()
        assert torch.equal(out, ref), frames
    _lib.poll_kernel_error()


def test_per_set_bank_write_lands_each_set_in_its_frame(dev):
    g = torch.Generator().manual_seed(5)
    h, w, cap_frames = 4, 6, 5
    hw = h * w
    halo = torch.zeros((SETS * PER, h + 2, w + 2, 640))
    halo[:, 1:-1, 1:-1] = torch.randn((SETS * PER, h, w, 640), generator=g)
    halo = halo.to(dev)
    bk = torch.full((SETS * PER, cap_frames * hw, 128), -5.0, device=dev)
    bv = torch.full((SETS * PER, cap_frames * hw, 512), -5.0, device=dev)
    frames = [3, 0, 4, 7]  # set 3: outside [0, t_max = 4]: writes nothing
    ops.bank_write_sets(halo, SETS * PER, SETS, h, w, 0, 128, bk, bv, cap_frames - 1,
                        torch.tensor(frames, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    want_k = torch.full_like(bk, -5.0)
    want_v = torch.full_like(bv, -5.0)
    interior = halo[:, 1:-1, 1:-1].reshape(SETS * PER, hw, 640)
    for s, t in enumerate(frames):
        if t < cap_frames:
            o = slice(s * PER, (s + 1) * PER)
            want_k[o, t * hw:(t + 1) * hw] = interior[o, :, :128]
            want_v[o, t * hw:(t + 1) * hw] = interior[o, :, 128:]
    assert torch.equal(bk, want_k) and torch.equal(bv, want_v)
