"""GPU: lock-step propagation of several clips as one batch (mivos_b200/lockstep.py) against the same
clips propagated one at a time.  The memory read is exact either way; the convolutions of a batch of
C*K maps may pick another split-K factor than those of K maps, i.e. another fp32 summation order (another
tile width alone gives the same bits: tests/test_gpu_conv_plans.py), so probabilities agree to the conv
tolerance of DESIGN.md §6 rather than bit for bit; bank bookkeeping is identical; the captured lock-step graph replays the eager launches bit for
bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mivos_b200  # noqa: E402
from mivos_b200 import _lib  # noqa: E402
from oracle import weights as Wt  # noqa: E402  (synthetic clips only)


def _clips(n, t, k, h=64, w=96):
    out = [Wt.synthetic_clip(t, h, w, k, seed=40 + i) for i in range(n)]
    return [o[0] for o in out], [o[1] for o in out]


def test_lockstep_equals_single_clip_passes(dev, nets):
    C, K, T = 3, 2, 7
    images, masks = _clips(C, T, K)
    net = nets[20]
    solo = []
    for i in range(C):
        core = mivos_b200.InferenceCore(net, None, images[i], K, mem_freq=2, device="cuda:0")
        solo.append((core.interact(masks[i], 2).copy(), core.prob.clone(), list(core.bank_trace)))
    cores = [mivos_b200.InferenceCore(net, None, images[i], K, mem_freq=2, device="cuda:0") for i in range(C)]
    steps = {"n": 0, "total": []}
    out = mivos_b200.LockstepSession(cores).interact(masks, 2, total_cb=lambda n: steps["total"].append(n),
                                                    step_cb=lambda: steps.__setitem__("n", steps["n"] + 1))
    _lib.poll_kernel_error()
    assert steps == {"n": T - 1, "total": [T - 1]}
    for i in range(C):
        m, p, tr = solo[i]
        assert cores[i].bank_trace == tr
        assert out[i].shape == m.shape and out[i].dtype == np.uint8
        d = (cores[i].prob - p).abs()
        assert float(d.max()) <= 3e-2 and float(d.mean()) <= 1e-3, (i, float(d.max()), float(d.mean()))
        assert float((out[i] != m).mean()) <= 1e-2
    # clips differ, so equal outputs across clips would mean the per-clip slices were mixed up
    assert float((cores[0].prob - cores[1].prob).abs().max()) > 0.1


def test_lockstep_second_interaction_fuses_per_clip(dev, nets):
    C, K, T = 2, 1, 6
    images, masks = _clips(C, T, K)
    net, fuse = nets[20], nets["fuse"]
    _, masks2 = _clips(C, T, K, h=64, w=96)
    masks2 = [m.flip(-1).contiguous() for m in masks2]
    solo = []
    for i in range(C):
        core = mivos_b200.InferenceCore(net, fuse, images[i], K, mem_freq=2, device="cuda:0")
        core.interact(masks[i], 0)
        solo.append((core.interact(masks2[i], 5).copy(), core.prob.clone(), list(core.bank_trace)))
    cores = [mivos_b200.InferenceCore(net, fuse, images[i], K, mem_freq=2, device="cuda:0") for i in range(C)]
    sess = mivos_b200.LockstepSession(cores)
    sess.interact(masks, 0)
    out = sess.interact(masks2, 5)  # backward pass bounded by frame 0 -> fuse_one_frame per clip
    _lib.poll_kernel_error()
    for i in range(C):
        m, p, tr = solo[i]
        assert cores[i].bank_trace == tr
        d = (cores[i].prob - p).abs()
        assert float(d.max()) <= 5e-2 and float(d.mean()) <= 2e-3, (i, float(d.max()), float(d.mean()))
        assert float((out[i] != m).mean()) <= 5e-2  # fused frames sit on the decision boundary (random FusionNet)
        assert cores[i].certain_mem_k.shape[2] == 2


def test_lockstep_graph_replay_is_bit_identical_to_eager(dev, nets, monkeypatch):
    C, K, T = 2, 2, 6
    images, masks = _clips(C, T, K)
    net = nets[20]
    res = []
    for graph in ("0", "1", "1"):  # eager, graph capture, cached graph replay
        monkeypatch.setenv("MIVOS_GRAPH", graph)
        if graph == "0":
            net.engine().__dict__.pop("_lock_steps", None)
        cores = [mivos_b200.InferenceCore(net, None, images[i], K, mem_freq=2, device="cuda:0") for i in range(C)]
        out = mivos_b200.LockstepSession(cores).interact(masks, 1)
        res.append(([o.copy() for o in out], [c.prob.clone() for c in cores]))
        if graph == "0":
            net.engine().__dict__.pop("_lock_steps", None)  # the eager step object must not serve the graph runs
    _lib.poll_kernel_error()
    for out, probs in res[1:]:
        for i in range(C):
            assert torch.equal(probs[i], res[0][1][i]) and (out[i] == res[0][0][i]).all()


def test_lockstep_rejects_mismatched_clips(dev, nets):
    images, masks = _clips(2, 5, 1)
    a = mivos_b200.InferenceCore(nets[20], None, images[0], 1, mem_freq=2, device="cuda:0")
    b = mivos_b200.InferenceCore(nets[20], None, images[1][:, :4], 1, mem_freq=2, device="cuda:0")
    with pytest.raises(mivos_b200._lib.MivosError):
        mivos_b200.LockstepSession([a, b])
    c = mivos_b200.InferenceCore(nets[50], None, images[1], 1, mem_freq=2, device="cuda:0")
    with pytest.raises(mivos_b200._lib.MivosError):
        mivos_b200.LockstepSession([a, c])  # another network object
