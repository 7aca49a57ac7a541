"""CPU: lock-step clips with their own pass plans (LockstepSession over clips of different length, mem_freq and
interaction history) — the per-set entry points' argument checks, the clip order and tick prefixes of
``schedule``, and the ragged host loop over the emulated C-ABI operators (tests/abi_emulator.py and, for the per-set
forms, tests/abi_emulator_sets.py) against each
clip's own InferenceCore.  The kernels, graphs and streams are covered on the GPU (tests/test_gpu_ragged_lockstep.py,
tests/test_gpu_memread_sets.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

import abi_emulator
import abi_emulator_sets


@pytest.fixture()
def rt(monkeypatch, prop_sd, fuse_sd):
    mv = abi_emulator.install_host_runtime(monkeypatch)
    abi_emulator_sets.install(monkeypatch, mv.ops)
    net = mv.PropagationNetwork(top_k=20, act_dtype=torch.float32)
    net.load_state_dict(prop_sd, strict=True)
    fuse = mv.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    return mv, net, fuse


def test_per_set_entry_points_validate_before_any_device_call():
    from mivos_b200 import _lib
    lib = _lib.load()
    null, p = C.c_void_p(0), C.c_void_p(256)
    before = lib.mivos_launch_count()
    for sets, counts, what in ((2, null, b"null count array"), (3, p, b"do not divide"), (0, p, b"do not divide")):
        assert lib.mivos_memory_read_sets(p, p, 64, 4, 32, p, 8, sets, 20, p, 1024, 0, 2, 4, null, null, p, 1 << 20, 0,
                                          counts, 0, null) == -1
        assert what in lib.mivos_last_error()
        assert lib.mivos_memory_read_dense_sets(p, p, 64, 4, 32, p, 8, sets, p, 1024, 0, 2, 4, p, 1 << 20, counts, 0,
                                                null) == -1
        assert what in lib.mivos_last_error()
        assert lib.mivos_memory_read_wide_sets(p, p, 64, 4, 128, p, 8, sets, 100, p, 1024, 0, 2, 4, null, null, p,
                                               1 << 20, counts, 0, null) == -1
        assert what in lib.mivos_last_error()
    assert lib.mivos_bank_write_sets(p, 4, 2, 2, 4, 640, 0, 128, p, p, 64, 7, null, null) == -1
    assert b"null frame array" in lib.mivos_last_error()
    assert lib.mivos_bank_write_sets(p, 4, 3, 2, 4, 640, 0, 128, p, p, 64, 7, p, null) == -1
    assert lib.mivos_bank_write_sets(p, 4, 2, 2, 4, 640, 0, 128, p, p, 64, 8, p, null) == -1  # frame 8 does not fit
    # the scalar-form checks still apply: top_k above the live bound, a bad output window
    assert lib.mivos_memory_read_sets(p, p, 64, 4, 16, p, 8, 2, 20, p, 1024, 0, 2, 4, null, null, p, 1 << 20, 0, p, 0,
                                      null) == -1
    assert lib.mivos_memory_read_sets(p, p, 64, 4, 32, p, 8, 2, 20, p, 1024, 768, 2, 4, null, null, p, 1 << 20, 0, p,
                                      0, null) == -1
    assert lib.mivos_launch_count() == before


@pytest.mark.parametrize("seed", range(6))
def test_clip_order_makes_active_and_memorizing_clips_prefixes(seed):
    from mivos_b200 import schedule
    rng = np.random.default_rng(seed)
    for forward in (True, False):
        plans = []
        for _ in range(int(rng.integers(2, 9))):
            t = int(rng.integers(2, 40))
            inter = set(int(x) for x in rng.integers(0, t, int(rng.integers(1, 4))))
            idx = sorted(inter)[int(rng.integers(0, len(inter)))]
            plans.append(schedule.plan_pass(t, inter, idx, forward, int(rng.integers(1, 6)), len(inter)))
        order = schedule.pass_order(plans)
        lens = [len(plans[c].frames) for c in order]
        assert lens == sorted(lens, reverse=True)
        assert order == sorted(range(len(plans)), key=lambda c: (-len(plans[c].frames), c))  # stable on ties
        for i in range(lens[0]):
            n, n_mem = schedule.tick_prefixes(plans, order, i)
            assert [c for c in order if len(plans[c].frames) > i] == order[:n]
            assert [c for c in order[:n] if plans[c].frames[i].memorize] == order[:n_mem]


# clip c: (length, mem_freq, first interaction, second interaction, third interaction or None)
CLIPS = [(7, 2, 2, 6, None), (9, 3, 4, 8, 1), (5, 1, 0, 0, None), (6, 2, 5, 2, None)]


def _ragged_setup(mv, net, fuse, K=2):
    from oracle import weights as Wt
    clips = [Wt.synthetic_clip(t, 64, 96, K, seed=60 + i) for i, (t, *_r) in enumerate(CLIPS)]
    mk = lambda: [mv.InferenceCore(net, fuse, img, K, mem_freq=CLIPS[i][1], device="cpu")  # noqa: E731
                  for i, (img, _m) in enumerate(clips)]
    return clips, mk


def _masks(clips, round_):
    return [m if round_ == 0 else (m.flip(-1) if round_ == 1 else m.flip(-2)).contiguous() for _img, m in clips]


def _run_both(mv, net, fuse):
    """Three interactions of the 4 CLIPS through one LockstepSession and through each clip's own InferenceCore."""
    clips, mk = _ragged_setup(mv, net, fuse)
    solo, cores = mk(), mk()
    sess = mv.LockstepSession(cores, ragged=True)
    rounds = []
    for r in range(3):
        idxs = [c[2 + r] if c[2 + r] is not None else c[2] for c in CLIPS]
        masks = _masks(clips, r)
        want = [s.interact(m, i) for s, m, i in zip(solo, masks, idxs)]
        got = sess.interact(masks, idxs)
        rounds.append((want, got))
    return solo, cores, rounds


def _compare(solo, cores, rounds):
    for want, got in rounds:
        for w, g in zip(want, got):
            assert (w == g).mean() >= 0.9999
    for s, c in zip(solo, cores):
        assert c.bank_trace == s.bank_trace
        d = (c.prob - s.prob).abs()
        assert float(d.max()) <= 1e-4
        assert c.certain_mem_k.shape == s.certain_mem_k.shape
        assert np.array_equal(c.np_masks, s.np_masks)


def test_ragged_session_equals_each_clips_own_interact(rt):
    mv, net, fuse = rt
    solo, cores, rounds = _run_both(mv, net, fuse)
    _compare(solo, cores, rounds)
    # the second round fuses on clips 0, 1, 3 (their passes are bounded by the first interaction), not on clip 2
    assert len(cores[1].interacted) == 3 and cores[2].interacted == {0}
    assert float((cores[0].prob[:, :5] - cores[3].prob[:, :5]).abs().max()) > 0.1  # clips were not mixed up


def test_ragged_session_callbacks_count_ticks(rt):
    from mivos_b200 import schedule
    mv, net, fuse = rt
    clips, mk = _ragged_setup(mv, net, fuse)
    cores = mk()
    calls = {"total": [], "steps": 0}
    idxs = [c[2] for c in CLIPS]
    mv.LockstepSession(cores, ragged=True).interact(_masks(clips, 0), idxs, total_cb=lambda n: calls["total"].append(n),
                                       step_cb=lambda: calls.__setitem__("steps", calls["steps"] + 1))
    ticks = sum(max(len(schedule.plan_pass(c.t, {i}, i, fw, c.mem_freq, 1).frames) for c, i in zip(cores, idxs))
                for fw in (True, False))
    assert calls == {"total": [ticks], "steps": ticks}


def test_ragged_comparison_has_teeth(rt, monkeypatch):
    """A read that gives every set the largest clip's count, or a bank write that puts every set in clip 0's frame,
    fails the comparison with the clips' own runs."""
    from mivos_b200 import ops
    mv, net, fuse = rt
    good_read, good_write = ops.memory_read_sets, ops.bank_write_sets

    def max_count_read(bank_k, bank_v, slots, qk, top_k, out, counts, **kw):
        return good_read(bank_k, bank_v, slots, qk, top_k, out, counts.max().expand(counts.shape).contiguous(), **kw)

    def clip0_frame_write(halo, k, sets, h, w, coff_k, coff_v, bank_k, bank_v, t_max, dyn_t):
        return good_write(halo, k, sets, h, w, coff_k, coff_v, bank_k, bank_v, t_max, dyn_t[:1].expand(dyn_t.shape).contiguous())

    for name, bad in (("memory_read_sets", max_count_read), ("bank_write_sets", clip0_frame_write)):
        with monkeypatch.context() as m:
            m.setattr(ops, name, bad)
            solo, cores, rounds = _run_both(mv, net, fuse)
            with pytest.raises(AssertionError):
                _compare(solo, cores, rounds)


def _recorder(monkeypatch, calls):
    """Records every emulated operator call: name, then per argument the shape and strides of a tensor or the value of
    a scalar (device pointers excluded)."""
    from mivos_b200 import ops

    def desc(v):
        if isinstance(v, torch.Tensor):
            return ("T", tuple(v.shape), v.stride(), v.dtype)
        if isinstance(v, (list, tuple)):
            return tuple(desc(x) for x in v)
        if hasattr(v, "cin_pad"):  # a packed convolution
            return ("conv", v.cin_pad, v.cout, v.taps)
        return v if isinstance(v, (int, float, bool, str, type(None))) else type(v).__name__

    for name in abi_emulator.OPS + abi_emulator_sets.OPS:
        f = getattr(ops, name)

        def wrap(*a, _n=name, _f=f, **k):
            vals = a
            if _n == "store_words":  # the pointer words change from run to run; their count does not
                vals = (a[0], len(list(a[1]))) + tuple(a[2:])
            calls.append((_n, tuple(desc(x) for x in vals), tuple(sorted((kk, desc(v)) for kk, v in k.items()))))
            return _f(*a, **k)
        monkeypatch.setattr(ops, name, wrap)


def test_same_plan_session_makes_the_operator_calls_of_one_plan(rt, monkeypatch, prop_sd, fuse_sd):
    """Clips that share one plan take the path the session always had: the calls of the one-plan loop (begin each
    interaction, run_pass forward and backward, finish), operator for operator, with the same shapes, strides and
    scalars — and no per-set form."""
    from oracle import weights as Wt
    from mivos_b200.inference_core import run_pass
    mv = rt[0]
    clips = [Wt.synthetic_clip(7, 64, 96, 2, seed=80 + i) for i in range(3)]
    calls = {}
    for mode in ("session", "one_plan"):
        net = mv.PropagationNetwork(top_k=20, act_dtype=torch.float32)  # fresh workspaces: the same allocations
        net.load_state_dict(prop_sd, strict=True)
        fuse = mv.FusionNet()
        fuse.load_state_dict(fuse_sd, strict=True)
        cores = [mv.InferenceCore(net, fuse, img, 2, mem_freq=2, device="cpu") for img, _ in clips]
        rec = calls[mode] = []
        with monkeypatch.context() as m:
            _recorder(m, rec)
            for idx, flip in ((2, False), (6, True)):
                masks = [(mk.flip(-1) if flip else mk).contiguous() for _, mk in clips]
                if mode == "session":
                    mv.LockstepSession(cores, ragged=True).interact(masks, idx)
                else:
                    keys = [c._begin_interaction(mk, idx)[0] for c, mk in zip(cores, masks)]
                    run_pass(cores, keys, idx, True)
                    run_pass(cores, keys, idx, False)
                    for c in cores:
                        c._finish_interaction()
    assert calls["session"] == calls["one_plan"] and len(calls["session"]) > 100
    assert not any(n.endswith("_sets") for n, _a, _k in calls["session"])


def test_prefix_ticks_allocate_no_workspace_beyond_the_full_batch(rt):
    from mivos_b200.frame_step import FrameStep
    mv, net, _ = rt
    Cn, K, H, W = 3, 2, 64, 96
    eng = net.engine()
    step = FrameStep(net, Cn, K, H, W, 16, ragged=True)
    step.bank_k.normal_()
    step.bank_v.normal_()
    states, batch = eng.new_query_states(H, W, Cn)
    eng.encode_query_batch(torch.randn((Cn, 3, H, W)), batch)
    frames = [torch.randn((1, 3, H, W)) for _ in range(Cn)]
    step.run_ragged(frames, states, [2, 2, 2], [2, 2, 2], Cn, [None] * Cn, [0] * Cn, graph=False)
    full = (eng.ws.bytes(), len(eng.ws._bufs))
    for n, n_mem in ((3, 2), (2, 2), (2, 0), (1, 1), (1, 0)):
        step.run_ragged(frames[:n], states[:n], [2] * n, [2] * n, n_mem, [None] * n, [0] * n, graph=False)
        assert (eng.ws.bytes(), len(eng.ws._bufs)) == full, (n, n_mem)


def test_ragged_sessions_take_clips_that_share_a_step(rt, prop_sd):
    """A ragged session takes clips of different length, mem_freq or history, and one interaction frame per clip; a
    session without ragged=True still refuses them.  Another object count, padded size or network, or more than 16
    objects, are refused either way."""
    from oracle import weights as Wt
    mv, net, _ = rt
    img, mask = Wt.synthetic_clip(5, 64, 96, 1, seed=1)
    a = mv.InferenceCore(net, None, img, 1, mem_freq=2, device="cpu")
    short = mv.InferenceCore(net, None, img[:, :4], 1, mem_freq=3, device="cpu")
    mv.LockstepSession([a, short], ragged=True)
    with pytest.raises(mv._lib.MivosError, match="ragged=True"):
        mv.LockstepSession([a, short])
    b = mv.InferenceCore(net, None, img, 1, mem_freq=2, device="cpu")
    with pytest.raises(mv._lib.MivosError, match="ragged=True"):
        mv.LockstepSession([a, b]).interact([mask, mask], [0, 1])
    img2, _ = Wt.synthetic_clip(5, 64, 96, 2, seed=1)
    img3, _ = Wt.synthetic_clip(5, 80, 96, 1, seed=1)
    other = mv.PropagationNetwork(top_k=20, act_dtype=torch.float32)
    other.load_state_dict(prop_sd, strict=True)
    img17, _ = Wt.synthetic_clip(3, 64, 96, 17, seed=9)
    for ragged in (False, True):
        with pytest.raises(mv._lib.MivosError, match="group the clips by object count"):
            mv.LockstepSession([a, mv.InferenceCore(net, None, img2, 2, mem_freq=2, device="cpu")], ragged=ragged)
        with pytest.raises(mv._lib.MivosError, match="padded size"):
            mv.LockstepSession([a, mv.InferenceCore(net, None, img3, 1, mem_freq=2, device="cpu")], ragged=ragged)
        with pytest.raises(mv._lib.MivosError, match="network"):
            mv.LockstepSession([a, mv.InferenceCore(other, None, img, 1, mem_freq=2, device="cpu")], ragged=ragged)
        with pytest.raises(mv._lib.MivosError, match="at most 16"):
            mv.LockstepSession([mv.InferenceCore(net, None, img17, 17, device="cpu") for _ in range(2)], ragged=ragged)
        with pytest.raises(mv._lib.MivosError, match="masks"):
            mv.LockstepSession([a, b], ragged=ragged).interact([mask], 0)
        with pytest.raises(mv._lib.MivosError, match="interaction frames"):
            mv.LockstepSession([a, b], ragged=ragged).interact([mask, mask], [0, 1, 2])
