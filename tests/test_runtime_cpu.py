"""CPU: the HOST runtime — InferenceCore (query-chunk cache, pass plan execution, bank writes, fusion
plumbing, argmax / unpad) and LockstepSession — running eagerly on CPU tensors over the emulated C-ABI
operators and a device-free stand-in for torch.cuda (tests/abi_emulator.py: test infrastructure; the
product's CUDA-device guard is replaced for these tests only).  Checked against the vectors the
UNMODIFIED reference produced (tests/golden/clip_lowres.npz) and against the oracle.  What this does
not cover — the kernels, CUDA graphs, streams — is covered on the GPU (tests/test_gpu_*.py)."""
import numpy as np
import pytest
import torch

import abi_emulator


@pytest.fixture()
def rt(monkeypatch, prop_sd, fuse_sd):
    mv = abi_emulator.install_host_runtime(monkeypatch)
    net = mv.PropagationNetwork(top_k=20, act_dtype=torch.float32)
    net.load_state_dict(prop_sd, strict=True)
    fuse = mv.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    return mv, net, fuse


def test_inference_core_host_runtime_matches_reference_golden(rt, golden):
    mv, net, fuse = rt
    g = golden("clip_lowres.npz")
    images = torch.from_numpy(g["images"])
    core = mv.InferenceCore(net, fuse, images, 2, mem_profile=0, mem_freq=2, device="cpu")
    calls = {"total": [], "steps": 0}
    m1 = core.interact(torch.from_numpy(g["mask"]), 0, total_cb=lambda n: calls["total"].append(n),
                       step_cb=lambda: calls.__setitem__("steps", calls["steps"] + 1))
    assert calls == {"total": [5], "steps": 5}
    assert m1.dtype == np.uint8 and m1.shape == (6, 64, 88) and tuple(core.pad) == (4, 4, 0, 0)
    assert core.bank_trace == [(1, 1), (2, 2), (3, 2), (4, 3), (5, 3)]
    d = (core.prob - torch.from_numpy(g["prob1"])).abs()
    assert float(d.max()) <= 3e-2 and float(d.mean()) <= 1e-3
    assert float((m1 != g["masks1"]).mean()) <= 0.01
    core.bank_trace = []
    m2 = core.interact(torch.from_numpy(g["mask2"]), 5)  # second interaction: fuse_one_frame on frames 1..4
    assert core.bank_trace == [(4, 2), (3, 3), (2, 3), (1, 4)]
    d = (core.prob - torch.from_numpy(g["prob2"])).abs()
    assert float(d.max()) <= 3e-2 and float(d.mean()) <= 1e-3
    assert float((m2 != g["masks2"]).mean()) <= 0.05
    assert core.certain_mem_k.shape == (2, 128, 2, 4, 6) and core.certain_mem_v.shape == (2, 512, 2, 4, 6)


@pytest.mark.parametrize("mem_profile", [1, 3])
def test_inference_core_host_clip_and_tiny_caches(rt, golden, mem_profile):
    """mem_profile >= 1: the clip stays on the host and frames are staged per use; mem_profile 3 also
    shrinks the query / image caches to one entry (wholesale flushes, reference :101-103,114-115)."""
    mv, net, _ = rt
    g = golden("clip_lowres.npz")
    core = mv.InferenceCore(net, None, torch.from_numpy(g["images"]), 2, mem_profile=mem_profile, mem_freq=2, device="cpu")
    m = core.interact(torch.from_numpy(g["mask"]), 0)
    assert core.bank_trace == [(1, 1), (2, 2), (3, 2), (4, 3), (5, 3)]
    assert float((core.prob - torch.from_numpy(g["prob1"])).abs().max()) <= 3e-2
    assert float((m != g["masks1"]).mean()) <= 0.01


def test_lockstep_session_equals_single_clip_passes(rt):
    from oracle import weights as Wt
    mv, net, fuse = rt
    C, K, T = 3, 2, 7
    clips = [Wt.synthetic_clip(T, 64, 96, K, seed=40 + i) for i in range(C)]
    clips2 = [c[1].flip(-1).contiguous() for c in clips]
    solo = []
    for img, mask in clips:
        core = mv.InferenceCore(net, fuse, img, K, mem_freq=2, device="cpu")
        core.interact(mask, 2)
        solo.append(core)
    cores = [mv.InferenceCore(net, fuse, img, K, mem_freq=2, device="cpu") for img, _ in clips]
    sess = mv.LockstepSession(cores)
    steps = {"n": 0, "total": []}
    out = sess.interact([m for _, m in clips], 2, total_cb=lambda n: steps["total"].append(n),
                        step_cb=lambda: steps.__setitem__("n", steps["n"] + 1))
    assert steps == {"n": T - 1, "total": [T - 1]}
    for i in range(C):
        assert cores[i].bank_trace == solo[i].bank_trace
        assert float((cores[i].prob - solo[i].prob).abs().max()) <= 1e-4, i
        assert (out[i] == solo[i].np_masks).mean() >= 0.9999
    assert float((cores[0].prob - cores[1].prob).abs().max()) > 0.1  # clips differ: slices were not mixed up
    # second interaction elsewhere: passes bounded by frame 2 -> per-clip fusion inside the lock-step loop
    for i in range(C):
        solo[i].bank_trace = []
        cores[i].bank_trace = []
        solo[i].interact(clips2[i], 6)
    out2 = sess.interact(clips2, 6)
    for i in range(C):
        assert cores[i].bank_trace == solo[i].bank_trace and len(cores[i].bank_trace) == 3
        assert float((cores[i].prob - solo[i].prob).abs().max()) <= 1e-4, i
        assert (out2[i] == solo[i].np_masks).mean() >= 0.9999
        assert cores[i].certain_mem_k.shape[2] == 2


def test_lockstep_session_of_one_clip_equals_interact(rt):
    """LockstepSession([core]) runs the single-clip step and pass loop: the same bits as core.interact, including a
    fused second interaction."""
    from oracle import weights as Wt
    mv, net, fuse = rt
    images, mask = Wt.synthetic_clip(7, 64, 96, 2, seed=44)
    solo = mv.InferenceCore(net, fuse, images, 2, mem_freq=2, device="cpu")
    core = mv.InferenceCore(net, fuse, images, 2, mem_freq=2, device="cpu")
    sess = mv.LockstepSession([core])
    for m, idx in ((mask, 2), (mask.flip(-1).contiguous(), 6)):
        want = solo.interact(m, idx)
        (got,) = sess.interact([m], idx)
        assert torch.equal(core.prob, solo.prob) and np.array_equal(got, want) and np.array_equal(core.np_masks, want)
        assert core.bank_trace == solo.bank_trace
    assert "_lock_steps" not in net.engine().__dict__  # one clip shares the single-clip steps


def test_frame_step_issues_the_same_operators_for_one_and_three_clips(rt, monkeypatch):
    """The step of C lock-step clips makes the launch sequence of one clip: the per-clip operators (memory read, skip
    broadcast, stem gather, aggregation, bank write) take the C clips as groups of one launch each."""
    import abi_emulator as E
    from mivos_b200 import ops
    from mivos_b200.frame_step import FrameStep
    mv, net, _ = rt
    names = []
    for name in E.OPS:
        monkeypatch.setattr(ops, name, lambda *a, _n=name, _f=getattr(ops, name), **k: (names.append(_n), _f(*a, **k))[1])
    K, H, W = 2, 64, 96
    eng = net.engine()
    seqs = {}
    for C in (1, 3):
        step = FrameStep(net, C, K, H, W, 16)
        step.bank_k.normal_()
        step.bank_v.normal_()
        states, batch = eng.new_query_states(H, W, C)
        eng.encode_query_batch(torch.randn((C, 3, H, W)), batch)
        frames = [torch.randn((1, 3, H, W)) for _ in range(C)]
        for memorize in (False, True):
            step.run(frames, states, 2, 2, memorize, graph=False)  # allocates the workspaces
            names.clear()
            step.run(frames, states, 2, 2, memorize, graph=False)
            seqs[C, memorize] = list(names)
    for memorize in (False, True):
        assert seqs[1, memorize] == seqs[3, memorize], memorize
        assert seqs[1, memorize].count("memory_read") == 1
    assert seqs[1, True].count("bank_write") == 1 and seqs[1, True].count("stem_gather") == 1


def test_a_dropped_network_releases_its_cached_steps(rt, prop_sd):
    """The frame steps cached on a network's engine do not keep the network alive: dropping it releases its
    workspaces, banks and graphs at once, not whenever the garbage collector next runs."""
    import gc
    import weakref
    from oracle import weights as Wt
    mv = rt[0]
    images, mask = Wt.synthetic_clip(4, 64, 96, 1, seed=3)
    gc.disable()
    try:
        net = mv.PropagationNetwork(top_k=20, act_dtype=torch.float32)
        net.load_state_dict(prop_sd, strict=True)
        cores = [mv.InferenceCore(net, None, images, 1, mem_freq=2, device="cpu") for _ in range(3)]
        cores[0].interact(mask, 1)
        mv.LockstepSession(cores[1:]).interact([mask, mask], 1)
        eng = weakref.ref(net.engine())
        assert eng().__dict__["_frame_steps"] and eng().__dict__["_lock_steps"]
        del net, cores
        assert eng() is None
    finally:
        gc.enable()


def test_lockstep_rejects_clips_that_cannot_share_a_plan(rt):
    from oracle import weights as Wt
    mv, net, _ = rt
    img, mask = Wt.synthetic_clip(5, 64, 96, 1, seed=1)
    a = mv.InferenceCore(net, None, img, 1, mem_freq=2, device="cpu")
    b = mv.InferenceCore(net, None, img[:, :4], 1, mem_freq=2, device="cpu")
    with pytest.raises(mv._lib.MivosError):
        mv.LockstepSession([a, b])
    c = mv.InferenceCore(net, None, img, 1, mem_freq=3, device="cpu")
    with pytest.raises(mv._lib.MivosError):
        mv.LockstepSession([a, c])
    with pytest.raises(mv._lib.MivosError):
        mv.LockstepSession([a, mv.InferenceCore(net, None, img, 1, mem_freq=2, device="cpu")]).interact([mask], 0)


def test_reference_layout_api_host_side(rt, golden):
    """PropagationNetwork's reference-layout methods (NCHW in / out: what generation/fusion_generator.py
    and a maintainer's own loop call) and FusionNet.forward over the emulated operators."""
    mv, net, fuse = rt
    g = golden("ops_lowres.npz")
    t = lambda k: torch.from_numpy(g[k])  # noqa: E731
    close = lambda a, b, tol=4e-3: float((a - b).abs().max()) <= tol * float(b.abs().max())  # noqa: E731
    f16, f8, f4, k16, v16 = net.get_query_values(t("frame"))
    assert close(f16, t("f16")) and close(f8[:, ::4], t("f8")) and close(f4[:, ::8], t("f4"))
    assert close(k16, t("k16")) and close(v16, t("v16"))
    mk, mv_ = net.memorize(t("frame"), t("mask")[1:])
    assert mk.shape == (2, 128, 1, 6, 8) and close(mk, t("mem_k")) and close(mv_, t("mem_v"))
    qv = net.get_query_values(t("frame3"))
    seg = net.segment_with_query(t("keys"), t("values"), *qv)
    assert float((seg - t("seg")).abs().max()) <= 3e-2
    at = net.get_attention(t("mem_k")[0:1], t("pos"), t("neg"), t("qk3"))
    assert close(at, t("attn"), 1e-5)
    fu = fuse(t("frame3"), t("seg")[0:1], t("agg")[1:2], t("attn"), t("dist"))
    assert close(fu, t("fuse"))


def test_attention_read_network_host_side(rt, golden, prop_sd):
    mv, _, _ = rt
    g = golden("attn_read.npz")
    net = mv.AttentionReadNetwork(act_dtype=torch.float32)
    net.load_state_dict(prop_sd, strict=False)  # fusion_model.py:187
    t = lambda k: torch.from_numpy(g[k])  # noqa: E731
    a1, a2 = net(t("image"), t("m11"), t("m21"), t("m12"), t("m22"), t("query"))
    for got, want in ((a1, t("attn1")), (a2, t("attn2"))):
        assert got.shape == want.shape
        assert float((got - want).abs().max()) <= 2e-2 * float(want.abs().max())


def test_s2m_network_and_controller_host_side(rt, golden):
    from oracle import weights
    mv, _, _ = rt
    net = mv.S2MNetwork(act_dtype=torch.float32)
    net.load_state_dict(weights.make_s2m_state_dict(), strict=True)
    g = golden("s2m_net.npz")
    ref = torch.from_numpy(g["logits"])
    assert float((net(torch.from_numpy(g["x"])) - ref).abs().max()) <= 5e-3 * float(ref.abs().max())
    c = golden("s2m_controller.npz")
    ctrl = mv.S2MController(net, int(c["k"]), ignore_class=255, device="cpu")
    m = ctrl.interact(torch.from_numpy(c["image"]), torch.from_numpy(c["prev"]), c["scr"])
    assert m.shape == c["mask"].shape
    assert float((m - torch.from_numpy(c["mask"])).abs().max()) <= 2e-2


def test_reset_gives_the_state_of_a_new_session(rt, golden):
    """InferenceCore.reset(): a reused core reproduces what a freshly constructed one computes — also after
    two interactions (certain memories, fused frames) and for a host-staged clip."""
    mv, net, fuse = rt
    g = golden("clip_lowres.npz")
    images, mask, mask2 = torch.from_numpy(g["images"]), torch.from_numpy(g["mask"]), torch.from_numpy(g["mask2"])
    for mem_profile in (0, 1):
        core = mv.InferenceCore(net, fuse, images, 2, mem_profile=mem_profile, mem_freq=2, device="cpu")
        m1 = core.interact(mask, 0).copy()
        p1 = core.prob.clone()
        core.interact(mask2, 5)
        core.reset()
        assert core.interacted == set() and core.certain_mem_k is None and core.query_buf == {} and core.bank_trace == []
        assert float(core.prob[1:].abs().max()) == 0 and float((core.prob[0] - 1e-7).abs().max()) == 0
        m1b = core.interact(mask, 0)
        assert core.bank_trace == [(1, 1), (2, 2), (3, 2), (4, 3), (5, 3)]
        assert torch.equal(core.prob, p1) and (m1b == m1).all()


def test_cfg1_480p_host_runtime_matches_reference_masks(rt, golden):
    """BASELINE configs[0] (480p 5-frame clip, 1 object, 3-frame memory) through the host runtime over
    the emulated operators: the DAVIS shape (854 -> 864 padding, 30x54 key maps, 1620-slot bank frames)."""
    from oracle import weights as Wt
    mv, _, _ = rt
    g = golden("cfg1_480p.npz")
    net = mv.PropagationNetwork(top_k=50, act_dtype=torch.float32)
    net.load_state_dict(Wt.make_prop_state_dict(1234), strict=True)
    images, mask = Wt.synthetic_clip(5, 480, 854, 1, seed=1234)
    core = mv.InferenceCore(net, None, images, 1, mem_profile=0, mem_freq=2, device="cpu")
    m = core.interact(mask, 0)
    assert m.shape == (5, 480, 854) and tuple(core.pad) == (5, 5, 0, 0) and (core.nh, core.nw) == (480, 864)
    assert core.bank_trace == [(1, 1), (2, 2), (3, 2), (4, 3)]
    assert float((m != g["masks"]).mean()) <= 1e-3
    d = (core.prob[:, :, :, ::8, ::8] - torch.from_numpy(g["prob_sub"])).abs()
    assert float(d.max()) <= 3e-2


def test_fusion_generator_client_host_side(rt, prop_sd):
    """SURVEY §8f-1 on the CPU: the FusionGenerator client flow (banks grown by torch.cat, reference-layout
    methods only) through our PropagationNetwork over the emulated operators vs the oracle."""
    import types
    from oracle import stm_oracle as O, weights as Wt
    from test_gpu_clients import fusion_generator_flow
    mv, _, _ = rt
    net = mv.PropagationNetwork(top_k=50, act_dtype=torch.float32)
    net.load_state_dict(prop_sd, strict=True)
    images, mask = Wt.synthetic_clip(5, 128, 168, 2, seed=31)
    soft = mask[1:] * 0.8 + 0.05
    ours = types.SimpleNamespace(pad_divide_by=mv.pad_divide_by, aggregate_wbg=mv.aggregate_wbg, memorize=net.memorize,
                                 get_query_values=net.get_query_values, segment_with_query=net.segment_with_query)
    orc = types.SimpleNamespace(pad_divide_by=O.pad_divide_by, aggregate_wbg=O.aggregate_wbg,
                                memorize=lambda f, m: O.memorize(prop_sd, f, m),
                                get_query_values=lambda f: O.get_query_values(prop_sd, f),
                                segment_with_query=lambda *a: O.segment_with_query(prop_sd, *a, top_k=50))
    d = (fusion_generator_flow(ours, images, soft, 2, 0, 4, mem_freq=2) - fusion_generator_flow(orc, images, soft, 2, 0, 4, mem_freq=2)).abs()
    assert float(d.max()) <= 3e-2 and float(d.mean()) <= 1e-3


def test_get_W_host_side(rt, golden):
    """PropagationNetwork.get_W (prop_net.py:183): [B,hw,hw] softmax over the memory axis, and the same
    affinity get_attention reduces (AttentionMemory.forward, prop_net.py:115-129)."""
    mv, net, _ = rt
    g = golden("ops_lowres.npz")
    mk16, qk = torch.from_numpy(g["mem_k"]), torch.from_numpy(g["qk3"])
    W = net.get_W(mk16, qk)
    B, hw = mk16.shape[0], qk.shape[-2] * qk.shape[-1]
    assert W.shape == (B, hw, hw)
    ref = torch.softmax(torch.bmm(mk16.reshape(B, 128, hw).transpose(1, 2), qk.reshape(1, 128, hw).expand(B, -1, -1) / 128 ** 0.5), dim=1)
    assert float((W - ref).abs().max()) <= 1e-6
    assert float((W.sum(1) - 1).abs().max()) <= 1e-5
