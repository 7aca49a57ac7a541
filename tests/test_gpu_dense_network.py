"""GPU: PropagationNetwork(top_k=None) — the reference's dense memory read (softmax over every bank slot,
prop_net.py:99-102) — through the drop-in surface, against the goldens of the UNMODIFIED reference
(oracle/gen_golden_dense.py), on the TF32 and the fp16 path, with the tolerances of tests/test_gpu_network.py:
probabilities max |dp| <= 3e-2, mean <= 1e-3; u8 masks <= 1 % (low res), <= 0.1 % (480p), fused frames <= 5 %;
bank bookkeeping exact."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mivos_b200  # noqa: E402
from mivos_b200 import _lib  # noqa: E402
from oracle import weights as Wt  # noqa: E402  (synthetic clips only)

P_MAX, P_MEAN = 3e-2, 1e-3


@pytest.fixture(scope="module", params=["tf32", "fp16"])
def dense(request, prop_sd, fuse_sd, dev):
    """top_k=None networks with the seeded weights, one per activation type, and FusionNet."""
    act = torch.float16 if request.param == "fp16" else torch.float32
    net = mivos_b200.PropagationNetwork(top_k=None, act_dtype=act)
    net.load_state_dict(prop_sd, strict=True)
    fuse = mivos_b200.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    return {"net": net.to(dev), "fuse": fuse.to(dev), "act": act}


def _close(p, ref):
    d = (torch.as_tensor(p).cpu() - torch.as_tensor(ref)).abs()
    assert float(d.max()) <= P_MAX and float(d.mean()) <= P_MEAN, (float(d.max()), float(d.mean()))


def test_dense_network_loads_the_state_dict(prop_sd):
    net = mivos_b200.PropagationNetwork(top_k=None)
    assert net.load_state_dict(prop_sd, strict=True) is not None and len(net.state_dict()) == 597
    assert net.top_k is None and net.memory.top_k is None and net.min_live_slots == 1


def test_segment_with_query_matches_reference(dev, dense, golden):
    live, g = golden("reference_live.npz"), golden("dense.npz")
    net = dense["net"]
    mk, mv = torch.from_numpy(live["ops_mk"]).to(dev), torch.from_numpy(live["ops_mv"]).to(dev)
    qv = [torch.from_numpy(live[f"ops_qv2_{i}"]).to(dev) for i in range(5)]
    _close(net.segment_with_query(mk, mv, *qv), g["seg_out"])
    _lib.poll_kernel_error()


def _clip_lowres():
    T, h, w, K = 6, 64, 88, 2
    images, mask = Wt.synthetic_clip(T, h, w, K, seed=21)
    _, mask2 = Wt.synthetic_clip(T, h, w, K, seed=22)
    return images, mask, torch.roll(mask2, shifts=(5, 9), dims=(2, 3))


def _traces(g, j):
    return [tuple(int(x) for x in r) for r in g[f"clip_trace{j}"]]


def test_clip_lowres_session_with_fusion(dev, dense, golden):
    g = golden("dense.npz")
    images, mask, mask2 = _clip_lowres()
    core = mivos_b200.InferenceCore(dense["net"], dense["fuse"], images, 2, mem_profile=0, mem_freq=2, device="cuda:0")
    m1 = core.interact(mask, 0)
    assert core.bank_trace == _traces(g, 1)
    _close(core.prob, g["clip_prob1"])
    assert float((m1 != g["clip_masks1"]).mean()) <= 0.01
    core.bank_trace = []
    m2 = core.interact(mask2, 5)  # second interaction: fuse_one_frame on frames 1..4
    assert core.bank_trace == _traces(g, 2)
    _close(core.prob, g["clip_prob2"])
    assert float((m2 != g["clip_masks2"]).mean()) <= 0.05
    pm = torch.zeros(3, 1, 64, 96)
    pm[2] = 1
    m3 = core.update_mask_only(pm, 2)
    assert (m3[2] == 2).all() and (m3[1] == m2[1]).all()
    _lib.poll_kernel_error()


def test_cfg1_480p_masks(dev, dense, golden):
    g = golden("dense.npz")
    images, mask = Wt.synthetic_clip(5, 480, 854, 1, seed=1234)
    for mem_profile in (0, 1):
        core = mivos_b200.InferenceCore(dense["net"], None, images, 1, mem_profile=mem_profile, mem_freq=2, device="cuda:0")
        m = core.interact(mask, 0)
        assert core.bank_trace == [(1, 1), (2, 2), (3, 2), (4, 3)]
        assert float((m != g["cfg1_masks"]).mean()) <= 1e-3
        d = (core.prob[:, :, :, ::8, ::8].cpu() - torch.from_numpy(g["cfg1_prob_sub"])).abs()
        assert float(d.max()) <= P_MAX
    _lib.poll_kernel_error()


@pytest.mark.parametrize("env", ["MIVOS_GRAPH", "MIVOS_BIDIR"])
def test_graph_replay_and_two_lanes_are_bit_identical(dev, dense, monkeypatch, env):
    """Captured graphs (device-side slot count) against eager launches, and the two-lane forward/backward overlap
    against one lane: the dense read's partition of the memory axis depends on hw alone, so the bits agree."""
    images, mask = Wt.synthetic_clip(9, 64, 96, 2, seed=11)
    res = []
    for on in (False, True, True):
        monkeypatch.setenv(env, "1" if on else "0")
        core = mivos_b200.InferenceCore(dense["net"], dense["fuse"], images, 2, mem_freq=2, device="cuda:0")
        m = core.interact(mask, 3)
        res.append((m.copy(), core.prob.clone(), list(core.bank_trace)))
    for m, p, tr in res[1:]:
        assert tr == res[0][2]
        assert torch.equal(p, res[0][1]) and (m == res[0][0]).all()
    _lib.poll_kernel_error()


def test_lockstep_session_equals_single_clip_passes(dev, dense):
    C, K, T = 4, 2, 7
    clips = [Wt.synthetic_clip(T, 64, 96, K, seed=40 + i) for i in range(C)]
    net = dense["net"]
    solo = []
    for img, m in clips:
        core = mivos_b200.InferenceCore(net, None, img, K, mem_freq=2, device="cuda:0")
        solo.append((core.interact(m, 2).copy(), core.prob.clone(), list(core.bank_trace)))
    cores = [mivos_b200.InferenceCore(net, None, img, K, mem_freq=2, device="cuda:0") for img, _ in clips]
    out = mivos_b200.LockstepSession(cores).interact([m for _, m in clips], 2)
    for i in range(C):
        m, p, tr = solo[i]
        assert cores[i].bank_trace == tr
        _close(cores[i].prob, p.cpu())
        assert float((out[i] != m).mean()) <= 1e-2
    _lib.poll_kernel_error()


def test_topk_network_unaffected_afterwards(dev, dense, nets, golden):
    """A top-k network used in the same process after a dense one still gives its usual results (engines are
    cached per top_k; the two reads keep separate workspaces)."""
    g = golden("clip_lowres.npz")
    core = mivos_b200.InferenceCore(nets[20], None, torch.from_numpy(g["images"]), 2, mem_profile=0, mem_freq=2,
                                    device="cuda:0")
    m1 = core.interact(torch.from_numpy(g["mask"]), 0)
    _close(core.prob, g["prob1"])
    assert float((m1 != g["masks1"]).mean()) <= 0.01
    assert nets[20].engine() is not dense["net"].engine() and nets[20].top_k == 20
    _lib.poll_kernel_error()
