"""GPU: PropagationNetwork(top_k=k) for 64 < k <= 1024 — the wide top-k read — through the drop-in surface, against
the goldens of the UNMODIFIED reference (oracle/gen_golden_wide.py), on the TF32 and the fp16 path, with the
tolerances of tests/test_gpu_network.py: probabilities max |dp| <= 3e-2, mean <= 1e-3; u8 masks <= 1 % (low res),
<= 0.1 % (480p), fused frames <= 5 %; bank bookkeeping exact."""
import pytest
import torch

pytestmark = pytest.mark.gpu

import mivos_b200  # noqa: E402
from mivos_b200 import _lib  # noqa: E402
from oracle import gen_golden_wide as GW  # noqa: E402  (input recipes of the goldens)
from oracle import weights as Wt  # noqa: E402  (synthetic clips only)

P_MAX, P_MEAN = 3e-2, 1e-3


@pytest.fixture(scope="module", params=["tf32", "fp16"])
def wide(request, prop_sd, fuse_sd, dev):
    """Networks with the seeded weights at the top_k of the goldens, one set per activation type, and FusionNet."""
    act = torch.float16 if request.param == "fp16" else torch.float32
    nets = {}
    for k in sorted({GW.SEG_TOP_K, GW.CLIP_TOP_K, GW.CFG1_TOP_K}):
        net = mivos_b200.PropagationNetwork(top_k=k, act_dtype=act)
        net.load_state_dict(prop_sd, strict=True)
        nets[k] = net.to(dev)
    fuse = mivos_b200.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    return {"nets": nets, "fuse": fuse.to(dev), "act": act}


def _close(p, ref):
    d = (torch.as_tensor(p).cpu() - torch.as_tensor(ref)).abs()
    assert float(d.max()) <= P_MAX and float(d.mean()) <= P_MEAN, (float(d.max()), float(d.mean()))


def _traces(g, j):
    return [tuple(int(x) for x in r) for r in g[f"clip_trace{j}"]]


def test_segment_with_query_matches_reference(dev, wide, golden):
    g = golden("wide.npz")
    mk, mv, qv = GW.seg_inputs(golden("reference_live.npz"))
    got = wide["nets"][GW.SEG_TOP_K].segment_with_query(mk.to(dev), mv.to(dev), *[t.to(dev) for t in qv])
    _close(got, g["seg_out"])
    _lib.poll_kernel_error()


def test_clip_session_with_fusion_matches_reference(dev, wide, golden):
    g = golden("wide.npz")
    images, mask, mask2 = GW.clip_inputs()
    T = images.shape[1]
    core = mivos_b200.InferenceCore(wide["nets"][GW.CLIP_TOP_K], wide["fuse"], images, 2, mem_profile=0, mem_freq=2,
                                    device="cuda:0")
    m1 = core.interact(mask, 0)
    assert core.bank_trace == _traces(g, 1)
    _close(core.prob, g["clip_prob1"])
    assert float((m1 != g["clip_masks1"]).mean()) <= 0.01
    core.bank_trace = []
    m2 = core.interact(mask2, T - 1)  # second interaction: fuse_one_frame on the frames between
    assert core.bank_trace == _traces(g, 2)
    _close(core.prob, g["clip_prob2"])
    assert float((m2 != g["clip_masks2"]).mean()) <= 0.05
    pm = torch.zeros(3, 1, images.shape[3], images.shape[4])
    pm[2] = 1
    m3 = core.update_mask_only(pm, 2)
    assert (m3[2] == 2).all() and (m3[1] == m2[1]).all()
    _lib.poll_kernel_error()


def test_cfg1_480p_masks(dev, wide, golden):
    g = golden("wide.npz")
    images, mask = Wt.synthetic_clip(5, 480, 854, 1, seed=1234)
    for mem_profile in (0, 1):  # device-resident clip and host-staged clip (pinned H2D per frame)
        core = mivos_b200.InferenceCore(wide["nets"][GW.CFG1_TOP_K], None, images, 1, mem_profile=mem_profile,
                                        mem_freq=2, device="cuda:0")
        m = core.interact(mask, 0)
        assert core.bank_trace == [(1, 1), (2, 2), (3, 2), (4, 3)]
        assert float((m != g["cfg1_masks"]).mean()) <= 1e-3
        d = (core.prob[:, :, :, ::8, ::8].cpu() - torch.from_numpy(g["cfg1_prob_sub"])).abs()
        assert float(d.max()) <= P_MAX
    _lib.poll_kernel_error()


@pytest.mark.parametrize("env", ["MIVOS_GRAPH", "MIVOS_BIDIR"])
def test_graph_replay_and_two_lanes_are_bit_identical(dev, wide, monkeypatch, env):
    """Captured graphs (device-side slot count) against eager launches, and the two-lane forward/backward overlap
    against one lane."""
    images, mask = Wt.synthetic_clip(9, 192, 256, 2, seed=11)
    res = []
    for on in (False, True, True):
        monkeypatch.setenv(env, "1" if on else "0")
        core = mivos_b200.InferenceCore(wide["nets"][GW.CLIP_TOP_K], wide["fuse"], images, 2, mem_freq=1,
                                        device="cuda:0")
        m = core.interact(mask, 3)
        res.append((m.copy(), core.prob.clone(), list(core.bank_trace)))
    for m, p, tr in res[1:]:
        assert tr == res[0][2]
        assert torch.equal(p, res[0][1]) and (m == res[0][0]).all()
    _lib.poll_kernel_error()


def test_lockstep_session_equals_single_clip_passes(dev, wide):
    C, K, T = 4, 2, 6
    clips = [Wt.synthetic_clip(T, 256, 320, K, seed=40 + i) for i in range(C)]  # 320 bank slots per frame
    net = wide["nets"][GW.CFG1_TOP_K]
    solo = []
    for img, m in clips:
        core = mivos_b200.InferenceCore(net, None, img, K, mem_freq=1, device="cuda:0")
        solo.append((core.interact(m, 2).copy(), core.prob.clone(), list(core.bank_trace)))
    cores = [mivos_b200.InferenceCore(net, None, img, K, mem_freq=1, device="cuda:0") for img, _ in clips]
    out = mivos_b200.LockstepSession(cores).interact([m for _, m in clips], 2)
    for i in range(C):
        m, p, tr = solo[i]
        assert cores[i].bank_trace == tr
        _close(cores[i].prob, p.cpu())
        assert float((out[i] != m).mean()) <= 1e-2
    _lib.poll_kernel_error()


def test_topk_50_network_unaffected_afterwards(dev, wide, nets, golden):
    """A top_k=50 network used in the same process after the wide ones still matches its goldens (engines are
    cached per top_k; the reads keep separate workspaces)."""
    g = golden("cfg1_480p.npz")
    images, mask = Wt.synthetic_clip(5, 480, 854, 1, seed=1234)
    core = mivos_b200.InferenceCore(nets[50], None, images, 1, mem_profile=0, mem_freq=2, device="cuda:0")
    m = core.interact(mask, 0)
    assert core.bank_trace == [(1, 1), (2, 2), (3, 2), (4, 3)]
    assert float((m != g["masks"]).mean()) <= 1e-3
    d = (core.prob[:, :, :, ::8, ::8].cpu() - torch.from_numpy(g["prob_sub"])).abs()
    assert float(d.max()) <= P_MAX
    assert nets[50].engine() is not wide["nets"][GW.CLIP_TOP_K].engine() and nets[50].top_k == 50
    _lib.poll_kernel_error()
