"""GPU: the drop-in surface (PropagationNetwork / FusionNet / InferenceCore) against the golden
fixtures generated from the UNMODIFIED reference and against the CPU oracle.

Stated fp32 tolerance (north_star): the convolution stacks run on the tensor cores in TF32
(10-bit-mantissa operands, fp32 accumulate, activations stored rounded-to-nearest TF32) while the
reference computes fp32, so
  * feature maps        : |d| <= 4e-3 * max|ref|          (bound of the fp16 / TF32 operand rounding)
  * probabilities       : max |dp| <= 3e-2, mean |dp| <= 1e-3   (measured 1.2e-2 / 1.4e-4)
  * u8 masks            : <= 1 % of pixels differ at low res with random weights, <= 0.1 % at
                          480p (measured 1e-5); fused frames sit on the decision boundary by
                          construction (random FusionNet) and are bounded by <= 5 %.
The memory read itself is exact (see test_gpu_memread.py); bank bookkeeping is bit-exact."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mivos_b200  # noqa: E402
from mivos_b200 import _lib  # noqa: E402
from oracle import stm_oracle as O, weights as Wt  # noqa: E402  (checker only)

FEAT_TOL, P_MAX, P_MEAN = 4e-3, 3e-2, 1e-3


def _feat_close(a, b, tol=FEAT_TOL):
    b = torch.as_tensor(b)
    a = a.detach().cpu()
    assert a.shape == b.shape
    assert float((a - b).abs().max()) <= tol * float(b.abs().max()), float((a - b).abs().max() / b.abs().max())


def test_query_values_and_memorize(dev, nets, golden):
    g = golden("ops_lowres.npz")
    net = nets[20]
    frame, mask = torch.from_numpy(g["frame"]).to(dev), torch.from_numpy(g["mask"]).to(dev)
    f16, f8, f4, k16, v16 = net.get_query_values(frame)
    assert f16.shape == (1, 1024, 6, 8) and f8.shape == (1, 512, 12, 16) and f4.shape == (1, 256, 24, 32)
    _feat_close(f16, g["f16"]); _feat_close(f8[:, ::4], g["f8"]); _feat_close(f4[:, ::8], g["f4"])
    _feat_close(k16, g["k16"]); _feat_close(v16, g["v16"])
    mk, mv = net.memorize(frame, mask[1:])
    assert mk.shape == (2, 128, 1, 6, 8) and mv.shape == (2, 512, 1, 6, 8)
    _feat_close(mk, g["mem_k"]); _feat_close(mv, g["mem_v"])
    _lib.poll_kernel_error()


def test_segment_attention_fusion(dev, nets, golden, prop_sd):
    g = golden("ops_lowres.npz")
    net, fuse = nets[20], nets["fuse"]
    keys, values = torch.from_numpy(g["keys"]).to(dev), torch.from_numpy(g["values"]).to(dev)
    # reference-layout entry point fed with the ORACLE's query features: isolates read + decoder
    qv = [t.to(dev) for t in O.get_query_values(prop_sd, torch.from_numpy(g["frame3"]))]
    seg = net.segment_with_query(keys, values, *qv).cpu()
    ref = torch.from_numpy(g["seg"])
    assert seg.shape == ref.shape
    assert float((seg - ref).abs().max()) <= P_MAX and float((seg - ref).abs().mean()) <= P_MEAN
    agg = mivos_b200.aggregate_wbg(ref.to(dev), keep_bg=True).cpu()
    assert float((agg - torch.from_numpy(g["agg"])).abs().max()) <= 1e-6
    at = net.get_attention(torch.from_numpy(g["mem_k"][0:1]).to(dev), torch.from_numpy(g["pos"]).to(dev),
                           torch.from_numpy(g["neg"]).to(dev), torch.from_numpy(g["qk3"]).to(dev))
    _feat_close(at, g["attn"], 1e-5)
    fu = fuse(torch.from_numpy(g["frame3"]).to(dev), torch.from_numpy(g["seg"][0:1]).to(dev), torch.from_numpy(g["agg"][1:2]).to(dev),
              torch.from_numpy(g["attn"]).to(dev), torch.from_numpy(g["dist"]).to(dev))
    _feat_close(fu, g["fuse"])
    _lib.poll_kernel_error()


def test_inference_core_lowres_clip_with_fusion(dev, nets, golden):
    g = golden("clip_lowres.npz")
    images = torch.from_numpy(g["images"])  # CPU, unpadded 64x88 -> padded 64x96 inside
    core = mivos_b200.InferenceCore(nets[20], nets["fuse"], images, 2, mem_profile=0, mem_freq=2, device="cuda:0")
    calls = {"total": [], "steps": 0}
    m1 = core.interact(torch.from_numpy(g["mask"]), 0, total_cb=lambda n: calls["total"].append(n),
                       step_cb=lambda: calls.__setitem__("steps", calls["steps"] + 1))
    assert calls == {"total": [5], "steps": 5}  # callback contract of inference_core.py:247-253,197-198
    assert m1.dtype == np.uint8 and m1.shape == (6, 64, 88) and tuple(core.pad) == (4, 4, 0, 0)
    assert core.bank_trace == [(1, 1), (2, 2), (3, 2), (4, 3), (5, 3)]  # bit-exact bank bookkeeping
    p1 = core.prob.cpu()
    d = (p1 - torch.from_numpy(g["prob1"])).abs()
    assert float(d.max()) <= P_MAX and float(d.mean()) <= P_MEAN
    assert float((m1 != g["masks1"]).mean()) <= 0.01
    assert core.prob.shape == (3, 6, 1, 64, 96) and core.masks.shape == (6, 1, 64, 96) and core.masks.dtype == torch.uint8
    core.bank_trace = []
    m2 = core.interact(torch.from_numpy(g["mask2"]), 5)  # second interaction -> fuse_one_frame on frames 1..4
    assert core.bank_trace == [(4, 2), (3, 3), (2, 3), (1, 4)]
    d = (core.prob.cpu() - torch.from_numpy(g["prob2"])).abs()
    assert float(d.max()) <= P_MAX and float(d.mean()) <= P_MEAN
    assert float((m2 != g["masks2"]).mean()) <= 0.05
    assert core.certain_mem_k.shape == (2, 128, 2, 4, 6) and core.certain_mem_v.shape == (2, 512, 2, 4, 6)
    # update_mask_only (inference_core.py:273-292)
    pm = torch.zeros(3, 1, 64, 96)
    pm[2] = 1
    m3 = core.update_mask_only(pm, 2)
    assert (m3[2] == 2).all() and (m3[1] == m2[1]).all()
    _lib.poll_kernel_error()


def test_cfg1_480p_plumbing_matches_reference_masks(dev, nets, golden):
    """BASELINE configs[0]: 480p 5-frame clip, 1 object, 3-frame memory (mem_freq=2)."""
    g = golden("cfg1_480p.npz")
    images, mask = Wt.synthetic_clip(5, 480, 854, 1, seed=1234)
    for mem_profile in (0, 1):  # device-resident clip and host-staged clip (pinned H2D per frame)
        core = mivos_b200.InferenceCore(nets[50], None, images, 1, mem_profile=mem_profile, mem_freq=2, device="cuda:0")
        m = core.interact(mask, 0)
        assert m.shape == (5, 480, 854) and tuple(core.pad) == (5, 5, 0, 0) and (core.nh, core.nw) == (480, 864)
        assert core.bank_trace == [(1, 1), (2, 2), (3, 2), (4, 3)]
        assert float((m != g["masks"]).mean()) <= 1e-3
        d = (core.prob[:, :, :, ::8, ::8].cpu() - torch.from_numpy(g["prob_sub"])).abs()
        assert float(d.max()) <= P_MAX
    _lib.poll_kernel_error()


def test_three_objects_against_oracle(dev, nets, prop_sd):
    """K=3 (cfg-3 shape at reduced resolution): 'others' mask channel, per-object reads, aggregation."""
    images, mask = Wt.synthetic_clip(4, 64, 96, 3, seed=5)
    core = mivos_b200.InferenceCore(nets[20], None, images, 3, mem_freq=1, device="cuda:0")
    m = core.interact(mask, 1)  # interaction in the middle: forward and backward passes
    oc = O.OracleInferenceCore(prop_sd, None, images, 3, mem_freq=1, top_k=20)
    om = oc.interact(mask, 1)
    assert core.bank_trace == oc.bank_trace
    d = (core.prob.cpu() - oc.prob).abs()
    assert float(d.max()) <= P_MAX and float(d.mean()) <= P_MEAN
    assert float((m != om).mean()) <= 0.01


def test_graph_replay_is_bit_identical_to_eager(dev, nets):
    """The captured per-frame CUDA graph (device-side bank counters, fixed launch geometry) must
    reproduce the step's eager launches bit for bit.  That a capacity-sized bank read through the device-side
    slot count gives what a read of the live slots with a host count gives is checked per read in
    test_gpu_memread.py, test_gpu_memread_dense.py and test_gpu_memread_wide.py."""
    images, mask = Wt.synthetic_clip(9, 64, 96, 2, seed=11)
    res = []
    for use_graph in (False, True, True):  # second graph run exercises the cached graphs
        core = mivos_b200.InferenceCore(nets[20], None, images, 2, mem_freq=2, device="cuda:0")
        core.use_graph = use_graph
        m = core.interact(mask, 3)
        res.append((m.copy(), core.prob.clone(), list(core.bank_trace)))
    for m, p, tr in res[1:]:
        assert tr == res[0][2]
        assert torch.equal(p, res[0][1]) and (m == res[0][0]).all()
    _lib.poll_kernel_error()


def test_get_W_matches_attention_memory(dev, nets, golden):
    """get_W (prop_net.py:183 -> AttentionMemory.forward :115-129) vs the formula in float64, and consistency with
    get_attention: area-pooled masks @ W, bilinear x16, equals the fused attention-map kernel."""
    g = golden("ops_lowres.npz")
    net = nets[20]
    mk16, qk = torch.from_numpy(g["mem_k"]).to(dev), torch.from_numpy(g["qk3"]).to(dev)
    W = net.get_W(mk16, qk)
    B, hw = mk16.shape[0], qk.shape[-2] * qk.shape[-1]
    assert W.shape == (B, hw, hw)
    a = torch.bmm(mk16.double().reshape(B, 128, hw).transpose(1, 2), (qk.double().reshape(1, 128, hw) / (128 ** 0.5)).expand(B, -1, -1))
    ref = torch.softmax(a, dim=1)
    assert float((W.double() - ref).abs().max()) <= 5e-6
    pos, neg = torch.from_numpy(g["pos"]).to(dev), torch.from_numpy(g["neg"]).to(dev)
    h, w = qk.shape[-2:]
    pooled = [torch.nn.functional.interpolate(m, size=(h, w), mode="area").view(1, 1, hw) @ W[0:1] for m in (pos, neg)]
    am = torch.nn.functional.interpolate(torch.cat(pooled, 1).reshape(1, 2, h, w), size=pos.shape[-2:], mode="bilinear", align_corners=False)
    at = net.get_attention(mk16[0:1], pos, neg, qk)
    assert float((am - at).abs().max()) <= 1e-5
    _lib.poll_kernel_error()
