"""GPU: whole sessions above 720p against the CPU oracle (oracle/gen_golden_hires.py; tests/golden/hires_1080p*.npz,
s2m_1080p.npz), on both element types, and a 4K session.

  1080p  1080x1920 (padded to 1088x1920), K=2, top-k 50, 6 frames, interactions at frames 0 and 5: frames 1..4 of
         the second interaction are fused with the attention map at hw = 8160, above the resident attention kernel's
         6912 key pixels, so they run the streamed kernel.  Criteria of test_gpu_zzz_fullsize.py's cfg-4 case: bank
         trace identical, max / mean |dp|, the same label on every decided pixel.
  S2M    the controller at 1088x1920 with K=2: in fp32 the 6-channel stem is wider than the untiled gather takes
         (1376 px), so it runs the column-tiled one; fp16 rows fit up to 2760 px.  Tolerances of test_gpu_z_s2m.py's
         controller test.
  4K     2160x3840 (135x240 = 32400 key pixels), K=1, mem_profile=2, two interactions: the session completes, the
         probabilities lie in [0, 1] and sum to 1 per pixel, and the frames between the interactions are fused."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mivos_b200  # noqa: E402
from mivos_b200 import _lib, ops  # noqa: E402
from oracle import gen_golden_hires as GH, weights as Wt  # noqa: E402  (checker only: inputs shared with the generator)
from test_gpu_zzz_fullsize import M_FRAC_FUSED, _check, _drift, _net, _report  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden(name):
    from oracle import golden_io
    return golden_io.load(os.path.join(ROOT, "tests", "golden", f"{name}.npz"))


def _count(monkeypatch, name):
    calls = []
    fn = getattr(ops, name)

    def wrapped(*a, **k):
        calls.append(1)
        return fn(*a, **k)
    monkeypatch.setattr(ops, name, wrapped)
    return calls


@pytest.mark.parametrize("act", ["fp16", "tf32"])
def test_1080p_fusion_two_interactions(act, prop_sd, fuse_sd, dev, monkeypatch):
    g = _golden("hires_1080p")
    images, inter, K, top_k, mem_freq, _ = GH.build_clip()
    streamed = _count(monkeypatch, "attention_map_streamed")
    net = _net(prop_sd, dev, top_k, act)
    fuse = mivos_b200.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    core = mivos_b200.InferenceCore(net, fuse.to(dev), images, K, mem_freq=mem_freq, device=dev)
    masks = None
    for idx, m in inter:
        masks = core.interact(m.to(dev), idx)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    assert [tuple(x) for x in g["trace"].tolist()] == core.bank_trace
    g["prob_l"] = g["prob_l"].reshape(K + 1, *core.prob.shape[-2:])
    assert len(streamed) == K * 4  # frames 1..4, one map per object
    d = _drift(core.prob, masks, g)
    _report(f"hires_1080p_{act}", d)
    _check(d, m_frac=M_FRAC_FUSED)


@pytest.mark.parametrize("act", ["fp16", "tf32"])
def test_1080p_s2m_controller(act, dev, monkeypatch):
    from interact.s2m_controller import S2MController
    g = _golden("s2m_1080p")
    tiled = _count(monkeypatch, "stem_gather_frames_tiled")
    net = mivos_b200.S2MNetwork(act_dtype=torch.float16 if act == "fp16" else torch.float32)
    net.load_state_dict(Wt.make_s2m_state_dict(), strict=True)
    image, prev, scr, k = GH.build_s2m()
    m = S2MController(net.to(dev), k, ignore_class=255, device=dev).interact(image, prev, scr)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    assert len(tiled) == (1 if act == "tf32" else 0) and m.shape == (k, 1, 1088, 1920)  # fp16 rows fit up to 2760 px
    st = int(g["stride"])
    for got, ref in ((m[:, :, ::st, ::st].cpu(), torch.from_numpy(g["prob_s"]).float()),
                     (m[0, 0].cpu(), torch.from_numpy(g["prob_l"]).float())):
        err = float((got - ref).abs().max())
        flips = float(((got > 0.5) != (ref > 0.5)).float().mean())
        print(f"[hires] s2m 1080p {act}: max |dp| {err:.3e}, label flips {flips:.2e}")
        assert err <= 3e-2 and flips <= 1e-2, (err, flips)


def test_4k_session_smoke(prop_sd, fuse_sd, dev, monkeypatch):
    H, W, T, K = 2160, 3840, 4, 1
    images, mask0 = Wt.synthetic_clip(T, H, W, K, seed=2160)
    mask1 = GH.GF.second_mask(K, H, W, 78)
    streamed = _count(monkeypatch, "attention_map_streamed")
    net = _net(prop_sd, dev, 50, "fp16")
    fuse = mivos_b200.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    core = mivos_b200.InferenceCore(net, fuse.to(dev), images, K, mem_profile=2, mem_freq=5, device=dev)
    core.interact(mask0.to(dev), 0)
    masks = core.interact(mask1.to(dev), T - 1)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    assert masks.shape == (T, H, W) and masks.dtype == np.uint8
    assert len(streamed) == K * (T - 2)  # frames 1..T-2 fused at hw = 32400
    p = core.prob[:, :, 0].float()
    assert bool(torch.isfinite(p).all()) and float(p.min()) >= 0.0 and float(p.max()) <= 1.0
    s = float((p.sum(0) - 1).abs().max())
    print(f"[hires] 4K session: max |sum p - 1| = {s:.2e}")
    assert s <= 1e-5
