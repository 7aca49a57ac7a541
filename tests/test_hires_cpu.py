"""CPU: frames above the shared-memory limits of the resident attention kernel (hw > 6912 key pixels: 1080p pads to
68 x 120 = 8160) and of the untiled 6-channel stem gather (1378 px in fp32, 2762 px in fp16).

  * the new entry points validate their arguments before any CUDA call;
  * the host queries mivos_attention_plan / mivos_stem_frames_plan draw the boundary exactly where the resident
    kernels start refusing shapes (tests/test_abi_symbols.py pins those widths);
  * over the emulated operators (tests/abi_emulator.py) get_attention, get_W, the fused frames of InferenceCore and
    S2M call the existing operator up to the boundary and the streamed / tiled one beyond it."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import abi_emulator
from mivos_b200 import _lib, ops


def _plan_attention(hw):
    r = C.c_int(-1)
    assert _lib.load().mivos_attention_plan(hw, C.byref(r)) == 0
    return r.value


def _plan_stem(cin, w, f16):
    r = C.c_int(-1)
    assert _lib.load().mivos_stem_frames_plan(cin, w, f16, C.byref(r)) == 0
    return r.value


def test_new_entry_points_reject_bad_arguments_without_a_device():
    lib = _lib.load()
    null, one = C.c_void_p(0), C.c_void_p(16)
    before = int(lib.mivos_launch_count())
    r = C.c_int(0)
    assert lib.mivos_attention_plan(0, C.byref(r)) == -1 and b"attention_plan" in lib.mivos_last_error()
    assert lib.mivos_attention_plan(64, None) == -1
    assert lib.mivos_stem_frames_plan(4, 64, 0, C.byref(r)) == -1 and b"3 or 6" in lib.mivos_last_error()
    assert lib.mivos_stem_frames_plan(6, 63, 0, C.byref(r)) == -1
    assert lib.mivos_stem_frames_plan(6, 0, 0, C.byref(r)) == -1
    assert lib.mivos_stem_frames_plan(6, 64, 0, None) == -1
    for args in ((null, one, 68, 120, one, one, one, one), (one, one, 68, 120, one, one, null, one),
                 (one, one, 68, 120, one, one, one, null), (C.c_void_p(20), one, 68, 120, one, one, one, one),
                 (one, one, 0, 120, one, one, one, one), (one, one, -1, -1, one, one, one, one),
                 (one, one, 1 << 15, 1 << 15, one, one, one, one)):
        assert lib.mivos_attention_map_streamed(*args, null) == -1, args
        assert b"attention_map_streamed" in lib.mivos_last_error()
    for args in ((null, one, 8160, one, one), (one, one, 8160, null, one), (one, one, 8160, one, null),
                 (one, C.c_void_p(24), 8160, one, one), (one, one, 0, one, one), (one, one, -5, one, one)):
        assert lib.mivos_attention_weights_streamed(*args, null) == -1, args
        assert b"attention_weights_streamed" in lib.mivos_last_error()
    for args in ((null, 1, 1088, 1920, one, 320, 0), (one, 1, 1088, 1920, null, 320, 0),
                 (one, 1, 1087, 1920, one, 320, 0), (one, 1, 1088, 1921, one, 320, 0), (one, 0, 1088, 1920, one, 320, 0),
                 (one, 1, 1088, 1920, one, 288, 0), (one, 1, 1088, 1920, one, 300, 0), (one, 1, 1088, 1920, C.c_void_p(8), 320, 0),
                 (one, 1, 0, 1920, one, 320, 1)):
        assert lib.mivos_stem_gather_frames_tiled(*args, null) == -1, args
        assert b"stem_gather_frames_tiled" in lib.mivos_last_error()
    assert int(lib.mivos_launch_count()) == before


def test_host_query_boundaries():
    assert _plan_attention(1) == 1 and _plan_attention(6912) == 1
    assert _plan_attention(6913) == 0 and _plan_attention(8160) == 0 and _plan_attention(32400) == 0
    # the widest frames mivos_stem_gather_frames admits, and the first it refuses (tests/test_abi_symbols.py)
    assert _plan_stem(6, 1376, 0) == 1 and _plan_stem(6, 1378, 0) == 0
    assert _plan_stem(6, 2760, 1) == 1 and _plan_stem(6, 2762, 1) == 0
    assert _plan_stem(3, 2760, 0) == 1 and _plan_stem(3, 2762, 0) == 0
    assert ops.attention_resident(6912) and not ops.attention_resident(6913)
    assert ops.stem_frames_untiled(6, 1376, False) and not ops.stem_frames_untiled(6, 1378, False)


# ------------------------------------------------------------------------------------------------ routing
def _recorder(monkeypatch, names):
    """Wrap the (emulated) operators `names` of ops so that every call is logged by name."""
    calls = []
    for name in names:
        fn = getattr(ops, name)

        def wrapped(*a, _fn=fn, _name=name, **k):
            calls.append(_name)
            return _fn(*a, **k)
        monkeypatch.setattr(ops, name, wrapped)
    return calls


def _stand_ins(monkeypatch):
    """The emulator plus stand-ins for the streamed / tiled operators (same header contracts as the resident ones)."""
    abi_emulator.install_host_runtime(monkeypatch)
    monkeypatch.setattr(ops, "attention_map_streamed", abi_emulator.attention_map)
    monkeypatch.setattr(ops, "attention_weights_streamed", abi_emulator.attention_weights)
    monkeypatch.setattr(ops, "stem_gather_frames_tiled", abi_emulator.stem_gather_frames)
    return _recorder(monkeypatch, ["attention_map", "attention_map_streamed", "attention_weights",
                                   "attention_weights_streamed", "stem_gather_frames", "stem_gather_frames_tiled"])


@pytest.fixture()
def net(monkeypatch, prop_sd):
    calls = _stand_ins(monkeypatch)
    import mivos_b200
    n = mivos_b200.PropagationNetwork(top_k=20, act_dtype=torch.float32)
    n.load_state_dict(prop_sd, strict=True)
    return n, calls


@pytest.mark.parametrize("h,w,streamed", [(64, 108, False), (31, 223, True), (68, 120, True)])
def test_get_attention_and_get_W_select_by_size(net, h, w, streamed):
    n, calls = net
    g = torch.Generator().manual_seed(h * w)
    hw = h * w
    mk = torch.randn(1, 128, 1, h, w, generator=g) * 0.05
    qk = torch.randn(1, 128, h, w, generator=g) * 0.05
    pos = torch.rand(1, 1, 16 * h, 16 * w, generator=g)
    neg = torch.rand(1, 1, 16 * h, 16 * w, generator=g)
    at = n.get_attention(mk[:, :, 0], pos, neg, qk)
    assert at.shape == (1, 2, 16 * h, 16 * w)
    assert calls == (["attention_map_streamed"] if streamed else ["attention_map"])
    calls.clear()
    W = n.get_W(mk, qk)
    assert W.shape == (1, hw, hw)
    assert calls == (["attention_weights_streamed"] if streamed else ["attention_weights"])
    # what get_attention reduces is the affinity get_W returns
    rows = torch.cat([F.avg_pool2d(m, 16).reshape(1, hw) for m in (pos, neg)]) @ W[0]
    want = F.interpolate(rows.reshape(1, 2, h, w), size=(16 * h, 16 * w), mode="bilinear", align_corners=False)
    assert float((at - want).abs().max()) <= 1e-4


def test_fused_frames_of_a_session_use_the_resident_kernel_at_small_sizes(net, fuse_sd):
    """A two-interaction session at 64 x 88 (hw = 24): the frames between the interactions are fused."""
    from oracle import weights as Wt
    import mivos_b200
    n, calls = net
    fuse = mivos_b200.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    img, mask = Wt.synthetic_clip(5, 64, 96, 2, seed=3)
    core = mivos_b200.InferenceCore(n, fuse, img, 2, mem_freq=2, device="cpu")
    core.interact(mask, 0)
    assert "attention_map" not in calls
    core.interact(mask.flip(-1).contiguous(), 4)
    assert calls.count("attention_map") == 2 * 3 and "attention_map_streamed" not in calls  # K = 2, frames 1..3


def test_fused_frame_above_the_resident_limit_uses_the_streamed_kernel(net, fuse_sd, monkeypatch):
    """InferenceCore.fuse_one_frame on a 496 x 3568 clip (31 x 223 = 6913 key pixels) — the call do_pass makes for
    every frame between two interactions, with the interacted frame's key in bank layout and the frame's query
    state.  The convolutions are shape-only stand-ins here: what is checked is which attention operator runs."""
    import mivos_b200
    n, calls = net
    monkeypatch.setattr(ops, "conv_gemm", lambda x, pc, nn_, h, w, out, **k: out)
    fuse = mivos_b200.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    H, W, K = 496, 3568, 2
    g = torch.Generator().manual_seed(5)
    img = torch.rand(1, 3, 3, H, W, generator=g)
    core = mivos_b200.InferenceCore(n, fuse, img, K, mem_freq=2, device="cpu")
    hw = (H // 16) * (W // 16)
    diff = torch.rand(K + 1, 1, H, W, generator=g) - 0.5
    core.pos_mask_diff, core.neg_mask_diff = diff.clamp(0, 1), (-diff).clamp(0, 1)
    qs = n.engine().new_query_state(H, W)
    qs.qk.copy_(torch.randn(hw, 128, generator=g) * 0.05)
    mk = torch.randn(K, hw, 128, generator=g) * 0.05
    masks = torch.rand(K + 1, 1, H, W, generator=g)
    out = core.fuse_one_frame(0, 2, 1, masks, masks, mk, qs)
    assert out.shape == (K + 1, 1, H, W)
    assert calls == ["attention_map_streamed"] * K


@pytest.mark.parametrize("W,f16,tiled", [(1376, False, False), (1392, False, True), (2752, True, False), (2768, True, True)])
def test_s2m_stem_selects_by_width(monkeypatch, W, f16, tiled):
    """S2M inputs are padded to multiples of 16: 1376 / 2752 px are the widest the untiled stem takes (fp32 / fp16)."""
    from mivos_b200 import engine
    from oracle import weights
    calls = _stand_ins(monkeypatch)
    monkeypatch.setattr(ops, "conv_gemm", lambda x, pc, nn_, h, w, out, **k: out)
    eng = engine.S2MEngine(weights.make_s2m_state_dict(), "cpu", act_dtype=torch.float16 if f16 else torch.float32)
    x = torch.rand(1, 6, 16, W, generator=torch.Generator().manual_seed(W))
    eng.logits_halo(x)
    assert calls == (["stem_gather_frames_tiled"] if tiled else ["stem_gather_frames"])
    stem = eng.ws.mat("stem", (16 // 2 + 2) * (W // 2 + 2), eng.pc["backbone.conv1"].cin_pad)
    want = abi_emulator.stem_gather_frames(x, torch.zeros(stem.shape, dtype=torch.float32))
    assert torch.equal(stem.float(), want.to(stem.dtype).float())
