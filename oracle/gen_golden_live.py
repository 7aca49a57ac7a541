"""Golden vectors of the original MiVOS modules on inputs that are NOT the other fixtures: what
tests/test_reference_live.py and tests/test_dropin_callers_cpu.py::test_iou_helpers_equal_the_reference compare the
oracle (and this repository's helpers) against.  Needs the original checkout (oracle/refshim.py):

  python -m oracle.gen_golden_live        -> tests/golden/reference_live.npz (+ parts, oracle/golden_io.py)
"""
from __future__ import annotations

import importlib
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden")

from oracle import golden_io, refshim, weights as Wt  # noqa: E402


def _np(t):
    return (t.detach().numpy() if torch.is_tensor(t) else np.asarray(t)).copy()  # a snapshot, not a view


def propagation_ops(r, prop_sd, fuse_sd, g):
    net, fuse = r.build_prop(prop_sd, top_k=20), r.build_fusion(fuse_sd)
    images, mask = Wt.synthetic_clip(3, 64, 96, 3, seed=2024)
    frame = images[:, 1]
    for i, t in enumerate(net.get_query_values(frame)):
        g[f"ops_qv{i}"] = _np(t)
    mk, mv = net.memorize(frame, mask[1:])
    g["ops_mk"], g["ops_mv"] = _np(mk), _np(mv)
    qv = net.get_query_values(images[:, 2])
    for i, t in enumerate(qv):
        g[f"ops_qv2_{i}"] = _np(t)
    seg = net.segment_with_query(mk, mv, *qv)
    g["ops_seg"] = _np(seg)
    agg = r.aggregate_wbg(seg, keep_bg=True)
    g["ops_agg"] = _np(agg)
    pos, neg = (mask[1:2] - seg[0:1]).clamp(0, 1), (seg[0:1] - mask[1:2]).clamp(0, 1)
    at = net.get_attention(mk[0:1], pos, neg, qv[3])
    g["ops_att"] = _np(at)
    g["ops_fuse"] = _np(fuse(images[:, 2], seg[0:1], agg[1:2], at, torch.tensor([[0.25, 0.75]])))


def inference_core(r, prop_sd, fuse_sd, g):
    images, mask = Wt.synthetic_clip(7, 64, 88, 2, seed=77)
    rc = r.InferenceCore(r.build_prop(prop_sd, top_k=20), r.build_fusion(fuse_sd), images, 2, mem_profile=0, mem_freq=2,
                         device="cpu")
    for j, (m, idx) in enumerate(((mask, 1), (mask.flip(-1).contiguous(), 6))):
        g[f"ic_masks{j}"] = _np(rc.interact(m, idx))
        g[f"ic_prob{j}"] = _np(rc.prob)
    g["ic_certain_mem_k"] = _np(rc.certain_mem_k)


def s2m(g):
    sd = Wt.make_s2m_state_dict()
    with refshim.reference_on_path():
        from interact.s2m_controller import S2MController
        from model.s2m.s2m_network import deeplabv3plus_resnet50 as S2M
        net = S2M().eval()
        net.load_state_dict(sd, strict=True)
        x = torch.randn((2, 6, 64, 80), generator=torch.Generator().manual_seed(5))
        g["s2m_logits"] = _np(net(x))
        image = torch.randn((1, 3, 64, 80), generator=torch.Generator().manual_seed(6))
        prev = torch.zeros((1, 64, 80), dtype=torch.int64)
        prev[:, 10:30, 10:40] = 1
        scr = np.full((60, 75), 255, dtype=np.uint8)
        scr[20:22, 5:50] = 1
        scr[40:42, 30:70] = 0
        g["s2m_ctrl"] = _np(S2MController(net, 1, ignore_class=255, device="cpu").interact(image, prev, scr))


def egress(g):
    from oracle.gen_golden_egress import load_reference_utils
    iu, pal = load_reference_utils()
    g["egress_palette"] = np.asarray(pal.pal_color_map())
    rng = np.random.default_rng(9)
    image = rng.integers(0, 256, size=(40, 52, 3), dtype=np.uint8)
    mask = (rng.integers(0, 7, size=(40, 52), dtype=np.uint8) * (rng.random((40, 52)) > 0.6)).astype(np.uint8)
    for j, alpha in enumerate((0.5, 0.37)):
        g[f"egress_overlay{j}"] = iu.overlay_davis(image, mask, alpha)
        g[f"egress_fade{j}"] = iu.overlay_davis_fade(image, mask, alpha)


def fusion_generator(r, prop_sd, g):
    images, mask = Wt.synthetic_clip(5, 128, 168, 2, seed=31)
    soft = mask[1:] * 0.8 + 0.05
    net = r.build_prop(prop_sd, top_k=50)
    with refshim.reference_on_path():
        FusionGenerator = importlib.import_module("generation.fusion_generator").FusionGenerator
        for k in [k for k in sys.modules if k == "generation" or k.startswith("generation.")]:
            sys.modules.pop(k)
    gen = FusionGenerator(net, images, mem_freq=2)
    gen.reset(2)
    g["fg_prob"] = _np(gen.interact_mask(soft, 2, 0, 4))


def attention_read(r, prop_sd, g):
    net = r.build_attn(prop_sd)
    gen = torch.Generator().manual_seed(123)
    image, query = torch.randn((1, 3, 48, 80), generator=gen), torch.randn((1, 3, 48, 80), generator=gen)
    m11, m21, m12, m22 = (torch.rand((1, 1, 48, 80), generator=gen) for _ in range(4))
    a1, a2 = net(image, m11, m21, m12, m22, query)
    g["attn_a1"], g["attn_a2"] = _np(a1), _np(a2)


def iou_helpers(g):
    with refshim.reference_on_path():
        spec = importlib.util.spec_from_file_location("_ref_util_tensor_util", os.path.join(refshim.REF_ROOT, "util", "tensor_util.py"))
        tu = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(tu)
    rng = np.random.default_rng(3)
    seg_np, gt_np = rng.random((40, 50)) > 0.5, rng.random((40, 50)) > 0.6
    seg_t, gt_t = torch.from_numpy(seg_np), torch.from_numpy(gt_np)
    g["iou_tensor_iu"] = np.stack([_np(x) for x in tu.compute_tensor_iu(seg_t, gt_t)])
    g["iou_tensor_iou"] = _np(tu.compute_tensor_iou(seg_t, gt_t))
    g["iou_np_iu"] = np.asarray(tu.compute_np_iu(seg_np, gt_np))
    g["iou_np_iou"] = np.asarray(tu.compute_np_iou(seg_np, gt_np))
    scores = torch.from_numpy(rng.random((4, 40, 50)).astype(np.float32))
    gt_soft = torch.from_numpy(rng.random((3, 1, 40, 50)).astype(np.float32))
    g["iou_multi_class"] = _np(tu.compute_multi_class_iou(scores, gt_soft))
    lab, lab2 = rng.integers(0, 4, (40, 50)), rng.integers(0, 4, (40, 50))
    g["iou_multi_class_idx"] = np.asarray(tu.compute_multi_class_iou_idx(lab, gt_soft[:, 0].numpy()))
    g["iou_multi_class_both_idx"] = np.asarray(tu.compute_multi_class_iou_both_idx(lab, lab2))


def main():
    torch.set_grad_enabled(False)
    prop_sd, fuse_sd = Wt.make_prop_state_dict(1234), Wt.make_fusion_state_dict(4321)  # tests/conftest.py
    g = {}
    r = refshim.load_reference()
    try:
        propagation_ops(r, prop_sd, fuse_sd, g)
        inference_core(r, prop_sd, fuse_sd, g)
        fusion_generator(r, prop_sd, g)
        attention_read(r, prop_sd, g)
        s2m(g)  # (constructed while the backbone download is patched out, like the networks above)
        egress(g)
        iou_helpers(g)
    finally:
        r._restore()
    files = golden_io.save(os.path.join(OUT, "reference_live.npz"), g)
    print(files, {k: v.shape for k, v in g.items()})


if __name__ == "__main__":
    main()
