"""GPU: one LockstepSession(ragged=True) over clips with their own pass plans — different length, mem_freq, first-interaction
frame, and a second interaction that fuses on some clips only — against each clip's own InferenceCore, on the
top-k, wide top-k and dense networks, in TF32 and fp16.  With the convolution plan pinned (one tile width, no split-K:
a batch of n*K maps then sums in the order of K maps) every clip gets the bits of its own run, which checks the
ragged bookkeeping exactly.  With the automatic plan, the batches of a tick — n*K maps for n = C down to 1 — may pick
other split-K factors than one clip's K maps, i.e. other fp32 summation orders, and the bank carries those
differences from frame to frame: the mean difference stays within the network tests' 1e-3, single pixels near a
top-k tie move by up to 0.085 (measured, TF32, 64x96), so the maximum is held to 0.1.  Bank bookkeeping is identical
either way, labels agree wherever the clip's own run decided them clearly, and the captured graphs replay the eager
launches bit for bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mivos_b200  # noqa: E402
from mivos_b200 import _lib  # noqa: E402
from oracle import weights as Wt  # noqa: E402  (synthetic clips only)

# clip: (length, mem_freq, first interaction, second interaction)
CLIPS = [(7, 2, 2, 6), (9, 3, 4, 8), (5, 1, 0, 0), (6, 2, 5, 2)]


def _clips(K, h, w):
    return [Wt.synthetic_clip(t, h, w, K, seed=70 + i) for i, (t, *_r) in enumerate(CLIPS)]


def _cores(net, fuse, clips, K):
    return [mivos_b200.InferenceCore(net, fuse, img, K, mem_freq=CLIPS[i][1], device="cuda:0")
            for i, (img, _m) in enumerate(clips)]


def _check(solo, cores, fused, tag):
    for i, (s, c) in enumerate(zip(solo, cores)):
        assert c.bank_trace == s.bank_trace, (tag, i)
        d = (c.prob - s.prob).abs()
        # fused frames run FusionNet on both sides of the decision boundary (random weights): the lock-step test's
        # fusion mean tolerance
        mx, mean = 1e-1, (2e-3 if fused else 1e-3)
        assert float(d.max()) <= mx and float(d.mean()) <= mean, (tag, i, float(d.max()), float(d.mean()))
        top2 = s.prob[:, :, 0].topk(2, dim=0).values
        decided = (top2[0] - top2[1]) > 2 * mx
        assert torch.equal(c.masks[:, 0][decided], s.masks[:, 0][decided]), (tag, i)


def _ragged(net, fuse, clips, K, rounds):
    solo, cores = _cores(net, fuse, clips, K), _cores(net, fuse, clips, K)
    sess = mivos_b200.LockstepSession(cores, ragged=True)
    for r in range(rounds):
        idxs = [c[2 + r] for c in CLIPS]
        masks = [(m if r == 0 else m.flip(-1)).contiguous() for _img, m in clips]
        for s, m, i in zip(solo, masks, idxs):
            s.interact(m, i)
        sess.interact(masks, idxs)
    _lib.poll_kernel_error()
    return solo, cores


def test_ragged_session_gives_each_clips_own_bits_under_a_pinned_conv_plan(dev, nets, monkeypatch):
    K = 2
    clips = _clips(K, 64, 96)
    monkeypatch.setenv("MIVOS_GRAPH", "0")  # eager: no graph captured under the pinned plan outlives this test
    lib = _lib.load()
    _lib.check(lib.mivos_conv_tile_override(32, 0), "mivos_conv_tile_override")
    try:
        solo, cores = _ragged(nets[20], nets["fuse"], clips, K, 2)
    finally:
        _lib.check(lib.mivos_conv_tile_override(0, 0), "mivos_conv_tile_override")
    for s, c in zip(solo, cores):
        assert c.bank_trace == s.bank_trace
        assert torch.equal(c.prob, s.prob) and torch.equal(c.masks, s.masks) and np.array_equal(c.np_masks, s.np_masks)


def test_ragged_session_equals_each_clips_own_run(dev, nets):
    K = 2
    clips = _clips(K, 64, 96)
    solo, cores = _ragged(nets[20], nets["fuse"], clips, K, 1)
    _check(solo, cores, False, "first")
    assert float((cores[0].prob[:, :5] - cores[3].prob[:, :5]).abs().max()) > 0.1  # clips were not mixed up


def test_ragged_session_fuses_a_second_interaction_on_some_clips(dev, nets):
    K = 1
    clips = _clips(K, 64, 96)
    solo, cores = _ragged(nets[20], nets["fuse"], clips, K, 2)
    _check(solo, cores, True, "second")
    assert [len(c.interacted) for c in cores] == [2, 2, 1, 2]


def test_ragged_graph_replay_is_bit_identical_to_eager(dev, nets, monkeypatch):
    K = 2
    clips = _clips(K, 64, 96)
    net = nets[20]
    res = []
    for graph in ("0", "1", "1"):  # eager, graph capture, cached graph replay
        monkeypatch.setenv("MIVOS_GRAPH", graph)
        if graph == "0":
            net.engine().__dict__.pop("_lock_steps", None)
        cores = _cores(net, nets["fuse"], clips, K)
        sess = mivos_b200.LockstepSession(cores, ragged=True)
        sess.interact([m for _i, m in clips], [c[2] for c in CLIPS])
        out = sess.interact([m.flip(-1).contiguous() for _i, m in clips], [c[3] for c in CLIPS])
        res.append(([o.copy() for o in out], [c.prob.clone() for c in cores]))
        if graph == "0":
            net.engine().__dict__.pop("_lock_steps", None)  # the eager step must not serve the graph runs
    _lib.poll_kernel_error()
    for out, probs in res[1:]:
        for i in range(len(CLIPS)):
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
def test_ragged_session_on_dense_and_wide_networks(dev, wide_dense_nets, top_k):
    K = 1
    clips = _clips(K, 160, 224)  # hw = 140: every read of the wide network has at least top_k live slots
    solo, cores = _ragged(wide_dense_nets[top_k], None, clips, K, 1)
    _check(solo, cores, False, f"top_k={top_k}")
