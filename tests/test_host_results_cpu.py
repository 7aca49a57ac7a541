"""CPU: a clip's results in host memory (InferenceCore(result_dev="cpu")).  The delivery entry point and the host
registration check their arguments before any CUDA call; over the emulated operators (tests/abi_emulator.py, and
tests/abi_emulator_host.py for the delivery) a host-results core matches the reference goldens and gives exactly
what a device-results core gives — single clips, a GUI-style edit sequence and lock-step sessions in any mix — and a
tick of device-result clips issues no delivery.  The kernel, graphs and streams are covered on the GPU
(tests/test_gpu_host_results.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

import abi_emulator
import abi_emulator_groups
import abi_emulator_host
import abi_emulator_sets
from mivos_b200 import _lib


@pytest.fixture()
def rt(monkeypatch, prop_sd, fuse_sd):
    mv = abi_emulator.install_host_runtime(monkeypatch)
    abi_emulator_sets.install(monkeypatch, mv.ops)
    abi_emulator_groups.install(monkeypatch, mv.ops)
    abi_emulator_host.install(monkeypatch, mv.ops)
    net = mv.PropagationNetwork(top_k=20, act_dtype=torch.float32)
    net.load_state_dict(prop_sd, strict=True)
    fuse = mv.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    return mv, net, fuse


def test_host_entry_points_validate_before_any_device_call():
    lib = _lib.load()
    null, p = C.c_void_p(0), C.c_void_p(256)
    before = lib.mivos_launch_count()
    for args in ((null, p, 1, 64, 96), (p, null, 1, 64, 96), (p, p, 0, 64, 96), (p, p, 65536, 64, 96),
                 (p, p, 1, 0, 96), (p, p, 1, 3, 5), (C.c_void_p(260), p, 1, 64, 96)):
        assert lib.mivos_deliver_planes(*args, null) == -1, args
        assert b"deliver_planes" in lib.mivos_last_error()
    dev = C.c_void_p(0)
    assert lib.mivos_host_register(null, 4096, C.byref(dev)) == -1
    assert lib.mivos_host_register(p, 0, C.byref(dev)) == -1
    assert lib.mivos_host_register(p, 4096, None) == -1
    assert lib.mivos_host_unregister(null) == -1
    assert b"host_unregister" in lib.mivos_last_error()
    assert lib.mivos_launch_count() == before


def test_result_dev_accepts_none_or_cpu_only(rt, golden):
    mv, net, _ = rt
    images = torch.from_numpy(golden("clip_lowres.npz")["images"])
    for bad in ("cuda", "cuda:0", torch.device("cuda:0"), "gpu", 1):
        with pytest.raises(mv._lib.MivosError):
            mv.InferenceCore(net, None, images, 2, device="cpu", result_dev=bad)
    for good in ("cpu", torch.device("cpu")):
        core = mv.InferenceCore(net, None, images, 2, device="cpu", result_dev=good)
        assert core.result_dev == torch.device("cpu")
        assert core.prob.shape == (3, 6, 1, 64, 96) and core.prob.dtype == torch.float32
        assert core.masks.shape == (6, 1, 64, 96) and core.masks.dtype == torch.uint8
        assert float(core.prob[1:].abs().max()) == 0 and bool((core.prob[0] == 1e-7).all())
        assert core._masks_unpadded is None and core._masks_host is None
    assert mv.InferenceCore(net, None, images, 2, device="cpu").result_dev == torch.device("cpu")  # the device here


def _assert_same(a, b):
    assert torch.equal(a.prob, b.prob)
    assert torch.equal(a.masks, b.masks)
    assert np.array_equal(a.np_masks, b.np_masks)
    assert a.bank_trace == b.bank_trace


@pytest.mark.parametrize("mem_profile", [0, 2, 3])
def test_host_results_match_the_goldens_and_device_results(rt, golden, mem_profile):
    """The reference's clip over two interactions (the second one fused), as the reference's own tests check it, and
    bit for bit what the same core with device results computes; the callbacks keep their rhythm."""
    mv, net, fuse = rt
    g = golden("clip_lowres.npz")
    images = torch.from_numpy(g["images"])
    cores = [mv.InferenceCore(net, fuse, images, 2, mem_profile=mem_profile, mem_freq=2, device="cpu", result_dev=r)
             for r in (None, "cpu")]
    calls = []
    for core in cores:
        c = {"total": [], "steps": 0}
        m1 = core.interact(torch.from_numpy(g["mask"]), 0, total_cb=lambda n: c["total"].append(n),
                           step_cb=lambda: c.__setitem__("steps", c["steps"] + 1))
        calls.append(c)
        assert core.bank_trace == [(1, 1), (2, 2), (3, 2), (4, 3), (5, 3)]
        d = (core.prob - torch.from_numpy(g["prob1"])).abs()
        assert float(d.max()) <= 3e-2 and float(d.mean()) <= 1e-3
        assert float((m1 != g["masks1"]).mean()) <= 0.01
    assert calls[0] == calls[1] == {"total": [5], "steps": 5}
    _assert_same(*cores)
    for core in cores:
        core.bank_trace = []
        m2 = core.interact(torch.from_numpy(g["mask2"]), 5)
        assert core.bank_trace == [(4, 2), (3, 3), (2, 3), (1, 4)]
        d = (core.prob - torch.from_numpy(g["prob2"])).abs()
        assert float(d.max()) <= 3e-2 and float(d.mean()) <= 1e-3
        assert float((m2 != g["masks2"]).mean()) <= 0.05
    _assert_same(*cores)
    # the label maps the deliveries keep are argmax(prob) of every frame
    host = cores[1]._host
    assert torch.equal(host.labels[:, 0], torch.argmax(cores[1].prob[:, :, 0], 0).to(torch.uint8))


def test_gui_sequence_gives_the_masks_of_device_results(rt, golden):
    """interact -> update_mask_only -> the caller clears masks[i] / np_masks[i] (interactive_gui.py:638-639) -> a
    second interaction with fusion: public masks and returned arrays agree with device results at every step."""
    mv, net, fuse = rt
    g = golden("clip_lowres.npz")
    images, mask, mask2 = torch.from_numpy(g["images"]), torch.from_numpy(g["mask"]), torch.from_numpy(g["mask2"])
    cores = [mv.InferenceCore(net, fuse, images, 2, mem_freq=2, device="cpu", result_dev=r) for r in (None, "cpu")]
    out = [[] for _ in cores]
    for core, o in zip(cores, out):
        o.append(core.interact(mask, 0).copy())
        o.append(core.update_mask_only(mv.pad_divide_by(mask2, 16, mask2.shape[-2:])[0], 3).copy())  # padded, as the GUI
        o.append(core.masks.clone())
        core.masks[2].zero_()
        core.np_masks[2].fill(0)
        o.append(core.interact(mask2, 5).copy())
        o.append(core.masks.clone())
    for a, b in zip(*out):
        assert (torch.equal(a, b) if isinstance(a, torch.Tensor) else np.array_equal(a, b))
    _assert_same(*cores)
    assert not np.array_equal(out[1][0][3], out[1][1][3])  # update_mask_only changed frame 3 of the public masks


def test_reset_refills_the_host_volumes(rt, golden):
    mv, net, fuse = rt
    g = golden("clip_lowres.npz")
    images, mask, mask2 = torch.from_numpy(g["images"]), torch.from_numpy(g["mask"]), torch.from_numpy(g["mask2"])
    core = mv.InferenceCore(net, fuse, images, 2, mem_freq=2, device="cpu", result_dev="cpu")
    m1 = core.interact(mask, 0).copy()
    p1 = core.prob.clone()
    core.interact(mask2, 5)
    prob, masks = core.prob, core.masks
    core.reset()
    assert core.prob is prob and core.masks is masks  # the same page-locked volumes
    assert float(core.prob[1:].abs().max()) == 0 and bool((core.prob[0] == 1e-7).all())
    assert int(core.masks.max()) == 0 and int(core._host.labels.max()) == 0 and int(core._host.labels_unpadded.max()) == 0
    assert torch.equal(core._host.labels_unpadded, torch.zeros_like(core._host.labels_unpadded))
    m1b = core.interact(mask, 0)
    assert torch.equal(core.prob, p1) and np.array_equal(m1b, m1)


def test_device_result_steps_issue_no_delivery(rt, golden):
    mv, net, fuse = rt
    g = golden("clip_lowres.npz")
    images = torch.from_numpy(g["images"])
    core = mv.InferenceCore(net, fuse, images, 2, mem_freq=2, device="cpu")
    core.interact(torch.from_numpy(g["mask"]), 0)
    core.interact(torch.from_numpy(g["mask2"]), 5)
    assert abi_emulator_host.DELIVERED == []
    host = mv.InferenceCore(net, fuse, images, 2, mem_freq=2, device="cpu", result_dev="cpu")
    host.interact(torch.from_numpy(g["mask"]), 0)
    # the interacted frame, then one per propagated frame (in the graph-captured step)
    assert abi_emulator_host.DELIVERED == [1] * 6
    abi_emulator_host.DELIVERED.clear()
    host.interact(torch.from_numpy(g["mask2"]), 5)
    assert abi_emulator_host.DELIVERED == [1] * 5  # frame 5, then the fused frames 4..1 delivered eagerly


# clip c: (length, mem_freq, object count, first interaction, second interaction)
CLIPS = [(7, 2, 2, 2, 6), (9, 3, 1, 4, 8), (5, 1, 3, 0, 0), (6, 2, 2, 5, 2)]


@pytest.mark.parametrize("kind", ["same_plan", "ragged", "mixed"])
@pytest.mark.parametrize("hosts", ["all", "half"])
def test_lockstep_sessions_with_host_results(rt, kind, hosts):
    """Same-plan, ragged and mixed-object sessions with every clip's results on the host, or every other clip's, give
    each clip the bits of the same session with device results; the ticks of a mixed session deliver the host
    clips of one tick with one launch."""
    from oracle import weights as Wt
    mv, net, fuse = rt
    if kind == "same_plan":
        spec = [(7, 2, 2, 2, 6)] * 3
    else:
        spec = [(t, f, k if kind == "mixed" else 2, a, b) for t, f, k, a, b in CLIPS]
    clips = [Wt.synthetic_clip(t, 64, 96, k, seed=90 + i) for i, (t, _f, k, _a, _b) in enumerate(spec)]
    host = [hosts == "all" or i % 2 == 1 for i in range(len(spec))]
    runs = []
    for use_host in (False, True):
        cores = [mv.InferenceCore(net, fuse, img, spec[i][2], mem_freq=spec[i][1], device="cpu",
                                  result_dev="cpu" if use_host and host[i] else None) for i, (img, _m) in enumerate(clips)]
        sess = mv.LockstepSession(cores, ragged=kind != "same_plan", mixed_objects=kind == "mixed")
        outs = []
        for r in range(2):
            masks = [m if r == 0 else m.flip(-1).contiguous() for _img, m in clips]
            idx = spec[0][3 + r] if kind == "same_plan" else [s[3 + r] for s in spec]
            outs.append(sess.interact(masks, idx))
        runs.append((cores, outs))
    (dcores, douts), (hcores, houts) = runs
    for a, b in zip(dcores, hcores):
        _assert_same(a, b)
    for da, ha in zip(douts, houts):
        assert all(np.array_equal(x, y) for x, y in zip(da, ha))
    assert [c._host is not None for c in hcores] == host
