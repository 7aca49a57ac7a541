"""CPU: lock-step clips with different object counts (LockstepSession(mixed_objects=True)).  The object-group entry
points (the *_groups forms of the memory reads, bank write, memorize stem, skip broadcast, v16 copy and decoder-tail
aggregation) check their arguments before any CUDA call; the mixed host loop over the emulated operators
(tests/abi_emulator.py, abi_emulator_sets.py and, for the group forms, abi_emulator_groups.py) gives each clip what
its own InferenceCore gives.  The kernels, graphs and streams are covered on the GPU (tests/test_gpu_mixed_objects.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

import abi_emulator
import abi_emulator_groups
import abi_emulator_sets
from mivos_b200 import _lib


def test_group_entry_points_validate_before_any_device_call():
    lib = _lib.load()
    null, p = C.c_void_p(0), C.c_void_p(256)
    before = lib.mivos_launch_count()

    def bad(rc, what):
        assert rc == -1
        assert what in lib.mivos_last_error(), lib.mivos_last_error()

    # reads: 4 objects over hw = 8 (2 x 4 halo), a bank of 64 slots
    for groups, first, counts, what in ((2, null, p, b"null group table"), (2, p, null, b"null count array"),
                                        (0, p, p, b"0 groups"), (5, p, p, b"5 groups")):
        bad(lib.mivos_memory_read_groups(p, p, 64, 4, 32, p, 8, groups, first, 20, p, 1024, 0, 2, 4, null, null, p,
                                         1 << 20, 0, counts, 0, null), what)
        bad(lib.mivos_memory_read_dense_groups(p, p, 64, 4, 32, p, 8, groups, first, p, 1024, 0, 2, 4, p, 1 << 20,
                                               counts, 0, null), what)
        bad(lib.mivos_memory_read_wide_groups(p, p, 64, 4, 128, p, 8, groups, first, 100, p, 1024, 0, 2, 4, null, null,
                                              p, 1 << 20, counts, 0, null), what)
    # the scalar-form checks still apply: top_k above the live bound, a bad output window, a null bank
    bad(lib.mivos_memory_read_groups(p, p, 64, 4, 16, p, 8, 2, p, 20, p, 1024, 0, 2, 4, null, null, p, 1 << 20, 0, p, 0,
                                     null), b"bad slot count")
    bad(lib.mivos_memory_read_groups(p, p, 64, 4, 32, p, 8, 2, p, 20, p, 1024, 768, 2, 4, null, null, p, 1 << 20, 0, p,
                                     0, null), b"output channel window")
    bad(lib.mivos_memory_read_dense_groups(null, p, 64, 4, 32, p, 8, 2, p, p, 1024, 0, 2, 4, p, 1 << 20, p, 0, null),
        b"null pointer")

    # bank write: 4 maps of 2 x 4 pixels into a bank of 64 slots (frames 0..7)
    bad(lib.mivos_bank_write_groups(p, 4, 2, p, 2, 4, 640, 0, 128, p, p, 64, 7, null, null), b"null frame array")
    bad(lib.mivos_bank_write_groups(p, 4, 2, null, 2, 4, 640, 0, 128, p, p, 64, 7, p, null), b"null group table")
    bad(lib.mivos_bank_write_groups(p, 4, 5, p, 2, 4, 640, 0, 128, p, p, 64, 7, p, null), b"5 groups for 4 maps")
    bad(lib.mivos_bank_write_groups(p, 4, 0, p, 2, 4, 640, 0, 128, p, p, 64, 7, p, null), b"0 groups for 4 maps")
    bad(lib.mivos_bank_write_groups(p, 4, 2, p, 2, 4, 640, 0, 128, p, p, 64, 8, p, null), b"does not fit capacity")

    # memorize stem: 4 maps of 16 x 16, kpad 80
    bad(lib.mivos_stem_gather_s2d_groups(p, p, 4, 2, null, 16, 16, p, 80, 1, 768, null), b"null group table")
    bad(lib.mivos_stem_gather_s2d_groups(p, null, 4, 2, p, 16, 16, p, 80, 1, 768, null), b"null pointer")
    bad(lib.mivos_stem_gather_s2d_groups(p, p, 4, 5, p, 16, 16, p, 80, 1, 768, null), b"5 groups for 4 maps")
    bad(lib.mivos_stem_gather_s2d_groups(p, p, 4, 0, p, 16, 16, p, 80, 1, 768, null), b"0 groups for 4 maps")
    bad(lib.mivos_stem_gather_s2d_groups(p, p, 4, 2, p, 15, 16, p, 80, 1, 768, null), b"must be even")
    bad(lib.mivos_stem_gather_s2d_groups(p, p, 4, 2, p, 16, 16, p, 64, 1, 768, null), b"kpad 64 too small")

    # skip broadcast and v16 copy: 4 images of 8 x 8, 64 channels
    bad(lib.mivos_upsample2x_add_groups(p, p, 4, 8, 8, 64, null, p, 2, null, 1, null), b"null group table")
    bad(lib.mivos_upsample2x_add_groups(p, p, 4, 8, 8, 64, null, null, 2, p, 1, null), b"bad arguments")
    bad(lib.mivos_upsample2x_add_groups(p, p, 4, 8, 8, 64, null, p, 5, p, 1, null), b"5 groups for 4 images")
    bad(lib.mivos_upsample2x_add_groups(p, p, 4, 8, 8, 64, null, p, 0, p, 1, null), b"0 groups for 4 images")
    bad(lib.mivos_halo_copy_groups(p, 2, null, 1024, 128, p, 1024, 512, 4, 8, 8, 512, 0, 1, 1, null),
        b"null group table")
    bad(lib.mivos_halo_copy_groups(null, 2, p, 1024, 128, p, 1024, 512, 4, 8, 8, 512, 0, 1, 1, null), b"null pointer")
    bad(lib.mivos_halo_copy_groups(p, 5, p, 1024, 128, p, 1024, 512, 4, 8, 8, 512, 0, 1, 1, null),
        b"5 groups for 4 images")
    bad(lib.mivos_halo_copy_groups(p, 2, p, 1024, 768, p, 1024, 512, 4, 8, 8, 512, 0, 1, 1, null),
        b"bad channel window")

    # decoder tail: 4 maps of 4 x 4 at 1/4 resolution
    bad(lib.mivos_upsample4x_sigmoid_aggregate_groups(p, 4, 2, null, 4, 4, 32, 0, null, p, null), b"null group table")
    bad(lib.mivos_upsample4x_sigmoid_aggregate_groups(p, 4, 2, p, 4, 4, 32, 0, null, null, null), b"null pointer")
    bad(lib.mivos_upsample4x_sigmoid_aggregate_groups(p, 4, 5, p, 4, 4, 32, 0, null, p, null), b"5 groups for 4 maps")
    bad(lib.mivos_upsample4x_sigmoid_aggregate_groups(p, 4, 0, p, 4, 4, 32, 0, null, p, null), b"0 groups for 4 maps")
    bad(lib.mivos_upsample4x_sigmoid_aggregate_groups(p, 33, 2, p, 4, 4, 32, 0, null, p, null),
        b"max 16 objects per group")
    bad(lib.mivos_upsample4x_sigmoid_aggregate_groups(p, 4, 2, p, 4, 4, 32, 32, null, p, null), b"bad shape")

    assert lib.mivos_launch_count() == before


@pytest.fixture()
def rt(monkeypatch, prop_sd, fuse_sd):
    mv = abi_emulator.install_host_runtime(monkeypatch)
    abi_emulator_sets.install(monkeypatch, mv.ops)
    abi_emulator_groups.install(monkeypatch, mv.ops)
    net = mv.PropagationNetwork(top_k=20, act_dtype=torch.float32)
    net.load_state_dict(prop_sd, strict=True)
    fuse = mv.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    return mv, net, fuse


# clip c: (objects, length, mem_freq, first interaction, second interaction)
CLIPS = [(1, 7, 2, 2, 6), (3, 9, 3, 4, 8), (2, 5, 1, 0, 0), (5, 6, 2, 5, 2)]


def _run_both(mv, net, fuse):
    """Two interactions of the 4 CLIPS through one mixed LockstepSession and through each clip's own InferenceCore;
    the second one fuses on the clips whose passes it bounds (0, 1, 3), not on clip 2."""
    from oracle import weights as Wt
    clips = [Wt.synthetic_clip(t, 64, 96, k, seed=90 + i) for i, (k, t, *_r) in enumerate(CLIPS)]
    mk = lambda: [mv.InferenceCore(net, fuse, img, CLIPS[i][0], mem_freq=CLIPS[i][2], device="cpu")  # noqa: E731
                  for i, (img, _m) in enumerate(clips)]
    solo, cores = mk(), mk()
    sess = mv.LockstepSession(cores, mixed_objects=True)
    rounds = []
    for r in range(2):
        idxs = [c[3 + r] for c in CLIPS]
        masks = [m if r == 0 else m.flip(-1).contiguous() for _img, m in clips]
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
        assert float((c.prob - s.prob).abs().max()) <= 1e-4
        assert np.array_equal(c.np_masks, s.np_masks)


def test_mixed_session_equals_each_clips_own_interact(rt):
    mv, net, fuse = rt
    solo, cores, rounds = _run_both(mv, net, fuse)
    _compare(solo, cores, rounds)
    assert len(cores[1].interacted) == 2 and cores[2].interacted == {0}


def test_mixed_comparison_has_teeth(rt, monkeypatch):
    """Each of these broken group operators fails the comparison with the clips' own runs: the aggregation reading
    the wrong group's range, the memorize stem's "others" summed across clips, the skip broadcast by uniform
    division, every group given the largest live count, every group written to the first clip's frame."""
    from mivos_b200 import ops
    import abi_emulator as E
    mv, net, fuse = rt
    good = {n: getattr(ops, n) for n in abi_emulator_groups.OPS}

    def shifted_aggregate(logits, n, h4, w4, first, coff=0, raw_out=None, prob_out=None):
        f = first.clone()
        f[1:-1] += 1  # every group boundary one map late
        return good["upsample4x_sigmoid_aggregate_groups"](logits, n, h4, w4, f, coff, raw_out, prob_out)

    def others_across_clips(frames, planes, n, first, out):
        H, W = frames.shape[-2:]
        rows = (H // 2 + 2) * (W // 2 + 2)
        f = [int(v) for v in first]
        objs = torch.cat([planes[f[g] + g + 1:f[g + 1] + g + 1] for g in range(len(f) - 1)])
        total = objs.sum(0, keepdim=True)
        for g in range(len(f) - 1):
            for i in range(f[g], f[g + 1]):
                x = torch.cat([frames[g:g + 1], objs[i:i + 1], total - objs[i:i + 1]], 1)
                E._stem_s2d_frames(x, out[i * rows:(i + 1) * rows])
        return out

    def uniform_skip(x, up, n, h, w, skip, first, x_relu=None):
        return E.upsample2x_add(x, up, n, h, w, x_relu=x_relu, skip=skip if n % skip.shape[0] == 0 else skip[:1])

    def max_count_read(bank_k, bank_v, slots, qk, top_k, out, counts, first, **kw):
        return good["memory_read_groups"](bank_k, bank_v, slots, qk, top_k, out,
                                          counts.max().expand(counts.shape).contiguous(), first, **kw)

    def clip0_frame_write(halo, n, h, w, coff_k, coff_v, bank_k, bank_v, t_max, dyn_t, first):
        return good["bank_write_groups"](halo, n, h, w, coff_k, coff_v, bank_k, bank_v, t_max,
                                         dyn_t[:1].expand(dyn_t.shape).contiguous(), first)

    for name, bad in (("upsample4x_sigmoid_aggregate_groups", shifted_aggregate),
                      ("stem_gather_groups", others_across_clips), ("upsample2x_add_groups", uniform_skip),
                      ("memory_read_groups", max_count_read), ("bank_write_groups", clip0_frame_write)):
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

    for name in abi_emulator.OPS + abi_emulator_sets.OPS + abi_emulator_groups.OPS:
        f = getattr(ops, name)

        def wrap(*a, _n=name, _f=f, **k):
            vals = a
            if _n == "store_words":  # the pointer words change from run to run; their count does not
                vals = (a[0], len(list(a[1]))) + tuple(a[2:])
            calls.append((_n, tuple(desc(x) for x in vals), tuple(sorted((kk, desc(v)) for kk, v in k.items()))))
            return _f(*a, **k)
        monkeypatch.setattr(ops, name, wrap)


def test_equal_object_counts_make_the_operator_calls_of_a_ragged_session(rt, monkeypatch, prop_sd, fuse_sd):
    from oracle import weights as Wt
    mv = rt[0]
    clips = [Wt.synthetic_clip(t, 64, 96, 2, seed=70 + i) for i, t in enumerate((7, 5, 6))]
    calls = {}
    for mode in ("mixed", "ragged"):
        net = mv.PropagationNetwork(top_k=20, act_dtype=torch.float32)  # fresh workspaces: the same allocations
        net.load_state_dict(prop_sd, strict=True)
        fuse = mv.FusionNet()
        fuse.load_state_dict(fuse_sd, strict=True)
        cores = [mv.InferenceCore(net, fuse, img, 2, mem_freq=f, device="cpu") for (img, _), f in zip(clips, (2, 3, 1))]
        rec = calls[mode] = []
        with monkeypatch.context() as m:
            _recorder(m, rec)
            sess = (mv.LockstepSession(cores, mixed_objects=True) if mode == "mixed"
                    else mv.LockstepSession(cores, ragged=True))
            for idxs in ([2, 1, 0], [6, 4, 3]):
                sess.interact([mk for _, mk in clips], idxs)
    assert calls["mixed"] == calls["ragged"] and len(calls["mixed"]) > 100
    assert not any(n.endswith("_groups") for n, _a, _k in calls["mixed"])


def test_prefix_ticks_allocate_no_workspace_beyond_the_full_batch(rt):
    from mivos_b200.frame_step import FrameStep
    mv, net, _ = rt
    ks, H, W = [3, 1, 2], 64, 96
    Cn = len(ks)
    eng = net.engine()
    step = FrameStep(net, Cn, max(ks), H, W, 16, ragged=True, maps=sum(ks))
    step.bank_k.normal_()
    step.bank_v.normal_()
    states, batch = eng.new_query_states(H, W, Cn)
    eng.encode_query_batch(torch.randn((Cn, 3, H, W)), batch)
    frames = [torch.randn((1, 3, H, W)) for _ in range(Cn)]
    step.run_ragged(frames, states, [2] * Cn, [2] * Cn, Cn, [None] * Cn, [0] * Cn, graph=False, ks=ks)
    full = (eng.ws.bytes(), len(eng.ws._bufs))
    for n, n_mem in ((3, 2), (2, 2), (2, 0), (1, 1), (1, 0)):
        step.run_ragged(frames[:n], states[:n], [2] * n, [2] * n, n_mem, [None] * n, [0] * n, graph=False, ks=ks)
        assert (eng.ws.bytes(), len(eng.ws._bufs)) == full, (n, n_mem)


def test_mixed_session_refusals(rt, prop_sd):
    """A mixed session takes clips of different object counts; it still refuses more than 16 objects, another padded
    size and another network — and a session without mixed_objects=True still refuses another object count."""
    from oracle import weights as Wt
    mv, net, _ = rt
    img, _ = Wt.synthetic_clip(5, 64, 96, 1, seed=1)
    img2, _ = Wt.synthetic_clip(5, 64, 96, 2, seed=1)
    a = mv.InferenceCore(net, None, img, 1, mem_freq=2, device="cpu")
    b = mv.InferenceCore(net, None, img2, 2, mem_freq=3, device="cpu")
    mv.LockstepSession([a, b], mixed_objects=True)
    with pytest.raises(mv._lib.MivosError, match="group the clips by object count"):
        mv.LockstepSession([a, b], ragged=True)
    img17, _ = Wt.synthetic_clip(3, 64, 96, 17, seed=9)
    with pytest.raises(mv._lib.MivosError, match="at most 16"):
        mv.LockstepSession([a, mv.InferenceCore(net, None, img17, 17, device="cpu")], mixed_objects=True)
    img3, _ = Wt.synthetic_clip(5, 80, 96, 1, seed=1)
    with pytest.raises(mv._lib.MivosError, match="padded size"):
        mv.LockstepSession([b, mv.InferenceCore(net, None, img3, 1, device="cpu")], mixed_objects=True)
    other = mv.PropagationNetwork(top_k=20, act_dtype=torch.float32)
    other.load_state_dict(prop_sd, strict=True)
    with pytest.raises(mv._lib.MivosError, match="network"):
        mv.LockstepSession([b, mv.InferenceCore(other, None, img, 1, device="cpu")], mixed_objects=True)
