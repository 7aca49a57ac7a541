"""GPU: a clip's results in page-locked host memory (InferenceCore(result_dev="cpu")).  The delivery kernel
(mivos_deliver_planes) against a host reference at ragged shapes, directly and from a replayed graph; single clips
and lock-step sessions with host results give the bits of device results (the same kernels compute them, only the
place the planes are written changes); the device memory of a host-results clip does not grow with its length."""
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mivos_b200  # noqa: E402
from mivos_b200 import _lib, ops, schedule  # noqa: E402
from mivos_b200.host_results import HostResults  # noqa: E402
from oracle import weights as Wt  # noqa: E402  (synthetic clips only)


@pytest.fixture(autouse=True)
def _clean_kernel_errors():
    yield
    _lib.poll_kernel_error()


# ---------------------------------------------------------------------- the kernel
@pytest.mark.parametrize("k1", [2, 17, 256])
def test_deliver_planes_at_ragged_shapes(dev, k1):
    """Clips of one padded size (64 x 112) with different h, w and pads, one with a null destination: planes byte-equal,
    labels torch.argmax (the first maximum) of the planes, padded and unpadded; nothing else of the volumes moves."""
    nh, nw, T = 64, 112, 5
    shapes = [((64, 112), (0, 0, 0, 0)), ((50, 101), (5, 6, 7, 7)), ((61, 97), (7, 8, 1, 2)), ((64, 100), (6, 6, 0, 0))]
    vols = [HostResults(k1, T, nh, nw, h, w, pad, dev) for (h, w), pad in shapes]
    g = torch.Generator(device=dev).manual_seed(k1)
    planes = (torch.randint(0, 4, (len(vols) * k1, 1, nh, nw), generator=g, device=dev) / 4).float()  # many ties
    planes += torch.rand(planes.shape, generator=g, device=dev) * (torch.rand(planes.shape, generator=g, device=dev) < 0.3)
    table = torch.zeros(len(vols) * ops.DELIVER_WORDS, dtype=torch.int64, device=dev)
    tis = [1, 4, 0, 2]
    words = []
    for c, v in enumerate(vols):
        words += v.record(tis[c], c * k1) if c != 2 else [0] * ops.DELIVER_WORDS  # clip 2: null destination
    ops.store_words(table, words)
    before = [v.prob.clone() for v in vols]
    ops.deliver_planes(planes, table, len(vols), nh, nw)
    torch.cuda.synchronize()
    ref = planes.cpu()
    for c, (v, ((h, w), pad)) in enumerate(zip(vols, shapes)):
        if c == 2:
            assert torch.equal(v.prob, before[c]) and int(v.labels.max()) == 0 and int(v.labels_unpadded.max()) == 0
            continue
        src = ref[c * k1:(c + 1) * k1]
        ti = tis[c]
        assert torch.equal(v.prob[:, ti].view(torch.int32), src.view(torch.int32)), c
        others = [t for t in range(T) if t != ti]
        assert torch.equal(v.prob[:, others], before[c][:, others])
        lab = torch.argmax(src[:, 0], 0).to(torch.uint8)
        assert torch.equal(v.labels[ti, 0], lab), c
        assert torch.equal(v.labels_unpadded[ti], lab[pad[2]:pad[2] + h, pad[0]:pad[0] + w]), c
        assert int(v.labels[others].max()) == 0 and int(v.labels_unpadded[others].max()) == 0


def test_deliver_planes_follows_the_table_in_a_replayed_graph(dev):
    """Captured once, the launch delivers to whatever frame and clip the table names when it is replayed."""
    nh, nw, T, k1 = 32, 48, 4, 3
    vols = [HostResults(k1, T, nh, nw, 30, 41, (3, 4, 1, 1), dev), HostResults(k1, T, nh, nw, 32, 48, (0, 0, 0, 0), dev)]
    planes = torch.rand((2 * k1, 1, nh, nw), device=dev)
    table = torch.zeros(2 * ops.DELIVER_WORDS, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.deliver_planes(planes, table, 2, nh, nw)
    for ti in range(T):
        ops.store_words(table, vols[0].record(ti, k1) + vols[1].record(T - 1 - ti, 0))
        planes.uniform_()
        graph.replay()
        torch.cuda.synchronize()
        p = planes.cpu()
        assert torch.equal(vols[0].prob[:, ti], p[k1:]) and torch.equal(vols[1].prob[:, T - 1 - ti], p[:k1])
        assert torch.equal(vols[0].labels[ti, 0], torch.argmax(p[k1:, 0], 0).to(torch.uint8))
        assert torch.equal(vols[0].labels_unpadded[ti], torch.argmax(p[k1:, 0], 0).to(torch.uint8)[1:31, 3:44])


# ---------------------------------------------------------------------- one clip
def _same(a, b, tag):
    assert torch.equal(a.prob.cpu(), b.prob.cpu()), tag
    assert torch.equal(a.masks.cpu(), b.masks.cpu()), tag
    assert np.array_equal(a.np_masks, b.np_masks), tag
    assert a.bank_trace == b.bank_trace, tag


def _session(core, images, mask, K):
    """A mid-clip first interaction (overlapped passes at mem_profile 0), a second one (fused frames), then the
    GUI-style sequence: update_mask_only, the caller clears masks[i] / np_masks[i], a third interaction with fusion.
    Returns every array handed back."""
    T, H, W = images.shape[1], images.shape[-2], images.shape[-1]
    m2 = Wt.synthetic_clip(T, H, W, K, seed=5)[1]
    m3 = mask.flip(-1).contiguous()
    out = [core.interact(mask, 3).copy(), core.interact(m2, T - 1).copy()]
    out.append(core.update_mask_only(mivos_b200.pad_divide_by(m3, 16, m3.shape[-2:])[0].to(core.device), 5).copy())
    core.masks[4].zero_()
    core.np_masks[4].fill(0)
    out.append(core.interact(m3, 0).copy())
    return out


@pytest.mark.parametrize("K", [1, 3, 17])
@pytest.mark.parametrize("mem_profile", [0, 2, 3])
def test_host_results_give_the_bits_of_device_results(dev, nets, K, mem_profile):
    images, mask = Wt.synthetic_clip(8, 64, 96, K, seed=20 + K)
    res = []
    for result_dev in (None, "cpu"):
        core = mivos_b200.InferenceCore(nets[20], nets["fuse"], images, K, mem_profile=mem_profile, mem_freq=2,
                                        device="cuda:0", result_dev=result_dev)
        res.append((core, _session(core, images, mask, K)))
    (dc, dout), (hc, hout) = res
    assert hc.prob.device.type == "cpu" and hc.masks.device.type == "cpu" and hc.result_dev == torch.device("cpu")
    _same(dc, hc, (nets["act"], K, mem_profile))
    for a, b in zip(dout, hout):
        assert np.array_equal(a, b)


def test_host_results_without_graphs(dev, nets, monkeypatch):
    monkeypatch.setenv("MIVOS_GRAPH", "0")
    K = 2
    images, mask = Wt.synthetic_clip(8, 64, 96, K, seed=31)
    cores = [mivos_b200.InferenceCore(nets[20], nets["fuse"], images, K, mem_freq=2, device="cuda:0", result_dev=r)
             for r in (None, "cpu")]
    outs = [_session(c, images, mask, K) for c in cores]
    _same(*cores, "eager")
    assert all(np.array_equal(a, b) for a, b in zip(*outs))


# ---------------------------------------------------------------------- lock-step sessions
# clip: (length, mem_freq, objects, first interaction, second interaction)
CLIPS = [(7, 2, 2, 2, 6), (9, 3, 1, 4, 8), (5, 1, 3, 0, 0), (6, 2, 2, 5, 2)]


@pytest.mark.parametrize("kind", ["same_plan", "ragged", "mixed"])
@pytest.mark.parametrize("hosts", ["all", "half"])
def test_lockstep_sessions_with_host_results(dev, nets, kind, hosts):
    spec = [(7, 2, 2, 2, 6)] * 3 if kind == "same_plan" else \
        [(t, f, k if kind == "mixed" else 2, a, b) for t, f, k, a, b in CLIPS]
    clips = [Wt.synthetic_clip(t, 64, 96, k, seed=50 + i) for i, (t, _f, k, _a, _b) in enumerate(spec)]
    host = [hosts == "all" or i % 2 == 1 for i in range(len(spec))]
    runs = []
    for use_host in (False, True):
        cores = [mivos_b200.InferenceCore(nets[20], nets["fuse"], img, spec[i][2], mem_freq=spec[i][1], device="cuda:0",
                                          result_dev="cpu" if use_host and host[i] else None)
                 for i, (img, _m) in enumerate(clips)]
        sess = mivos_b200.LockstepSession(cores, ragged=kind != "same_plan", mixed_objects=kind == "mixed")
        outs = []
        for r in range(2):
            masks = [(m if r == 0 else m.flip(-1)).contiguous() for _img, m in clips]
            outs.append(sess.interact(masks, spec[0][3 + r] if kind == "same_plan" else [s[3 + r] for s in spec]))
        runs.append((cores, outs))
    (dcores, douts), (hcores, houts) = runs
    for i, (a, b) in enumerate(zip(dcores, hcores)):
        _same(a, b, (kind, hosts, i))
    for da, ha in zip(douts, houts):
        assert all(np.array_equal(x, y) for x, y in zip(da, ha))


# ---------------------------------------------------------------------- device memory
def _peak(prop_sd, images, mask, K, result_dev):
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()  # what earlier tests still hold is not this run's
    torch.cuda.reset_peak_memory_stats()
    net = mivos_b200.PropagationNetwork(top_k=50, act_dtype=torch.float16)
    net.load_state_dict(prop_sd, strict=True)
    net = net.to("cuda:0")
    core = mivos_b200.InferenceCore(net, None, images, K, mem_profile=2, mem_freq=5, device="cuda:0",
                                    result_dev=result_dev)
    core.interact(mask, 0)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del core, net
    gc.collect()
    return peak


def test_host_results_device_memory_does_not_grow_with_clip_length(dev, prop_sd):
    """480p, K = 2, mem_profile 2: clips of 20 and 70 frames get the same 32-frame bank and the same query and image
    caches.  With host results the longer clip's peak is not higher; with device results the peaks grow by the 50
    frames' volume, probabilities and label maps, more than with host results.  (Under both settings the 20-frame
    clip's peak has been measured 242.5 MB above the 70-frame clip's on an H100; the cause is not known, so the two
    settings are compared with each other.)"""
    K, H, W = 2, 480, 854
    nh, nw = 480, 864
    assert {(schedule.bank_capacity_frames(t, 5, 1, 0) + 15) // 16 * 16 for t in (20, 70)} == {32}
    images, mask = Wt.synthetic_clip(70, H, W, K, seed=3)
    peaks = {}
    for rd in ("cpu", None):
        for t in (20, 70):
            peaks[rd, t] = _peak(prop_sd, images[:, :t].contiguous(), mask, K, rd)
    grow = (K + 1) * 50 * nh * nw * 4 + 50 * (nh * nw + H * W)
    host_diff = peaks["cpu", 70] - peaks["cpu", 20]
    print(f"peak device memory: host results {peaks['cpu', 20]} / {peaks['cpu', 70]} B (20 / 70 frames, difference "
          f"{host_diff} B); device results {peaks[None, 20]} / {peaks[None, 70]} B (difference "
          f"{peaks[None, 70] - peaks[None, 20]} B, the 50-frame volume is {grow} B)")
    # host results: the longer clip needs no more device memory than the shorter one
    assert host_diff <= 2 << 20
    # device results: at each length they hold the clip's volume on top of what host results hold, so from 20 to 70
    # frames they grow by the 50 frames' volume more than host results do (up to allocation rounding)
    assert (peaks[None, 70] - peaks["cpu", 70]) - (peaks[None, 20] - peaks["cpu", 20]) >= grow - (2 << 20)


def test_host_results_at_1080p(dev, nets):
    K = 2
    images, mask = Wt.synthetic_clip(5, 1080, 1920, K, seed=11)
    m2 = Wt.synthetic_clip(5, 1080, 1920, K, seed=12)[1]
    cores = [mivos_b200.InferenceCore(nets[50], nets["fuse"], images, K, mem_profile=2, device="cuda:0", result_dev=r)
             for r in (None, "cpu")]
    outs = [[c.interact(mask, 2).copy(), c.interact(m2, 4).copy()] for c in cores]
    assert cores[1].prob.shape == (K + 1, 5, 1, 1088, 1920)
    _same(*cores, "1080p")
    assert all(np.array_equal(a, b) for a, b in zip(*outs))
