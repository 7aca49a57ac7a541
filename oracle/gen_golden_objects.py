"""Golden vectors of the original MiVOS modules with MORE THAN 16 OBJECTS (the reference takes any count; the u8
label map caps it at 255).  Needs the original checkout (oracle/refshim.py):

  python -m oracle.gen_golden_objects    -> tests/golden/objects.npz (+ parts, oracle/golden_io.py), MANIFEST_objects.json

Contents:
  agg_K{K}_{mode}   model.aggregate on [K,1,9,13] probabilities regenerated from their seed (agg_inputs), K in
                    {17, 64, 255}, mode wbg_hard / wbg_soft / sbg (aggregate_wbg(keep_bg=True, hard=True),
                    aggregate_wbg(keep_bg=True), aggregate_sbg(keep_bg=True))
  clip{K}_*         InferenceCore(top_k=50) over CLIPS[K] (clip_inputs): two interactions, on the first and the last
                    frame, so that the second one fuses the frames between; u8 masks of both, the probability volume
                    after each at a stride of 4 pixels (prob_sub), and the bank trace of each
The oracle-vs-reference differences go to MANIFEST_objects.json (0.0 expected, as for the other goldens).
"""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden")

from oracle import golden_io, refshim, stm_oracle as O, weights as Wt  # noqa: E402

AGG_K = (17, 64, 255)
AGG_HW = (9, 13)
# K -> (frames, height, width, top_k, mem_freq).  At 64 x 96 a bank frame holds 4 * 6 = 24 slots, so the K = 255
# clip reads its top 20 (top_k 50 would fail the live-slot rule on the first frame, in the reference too).
CLIPS = {17: (8, 112, 176, 50, 2), 40: (10, 112, 176, 50, 2), 255: (4, 64, 96, 20, 2)}
SUB = 4  # stride of the stored probability samples


def _np(t):
    return (t.detach().numpy() if torch.is_tensor(t) else np.asarray(t)).copy()


def _diff(a, b) -> float:
    return float((torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max())


def agg_inputs(K):
    """Probabilities in (0, 1) with a few pixels at the clamp limits (0 and 1 exactly)."""
    g = torch.Generator().manual_seed(9000 + K)
    p = torch.rand((K, 1) + AGG_HW, generator=g)
    p[:, 0, 0, 0] = 0.0
    p[:, 0, 0, 1] = 1.0
    p[K // 2, 0, 1, :] = 1.0
    return p.contiguous()


def clip_inputs(K):
    T, h, w, _, _ = CLIPS[K]
    images, mask = Wt.synthetic_clip(T, h, w, K, seed=300 + K)
    _, mask2 = Wt.synthetic_clip(T, h, w, K, seed=400 + K)
    return images, mask, torch.roll(mask2, shifts=(3, 7), dims=(2, 3))


def aggregate(ref, g, report):
    for K in AGG_K:
        p = agg_inputs(K)
        for mode, fn, o_fn in (("wbg_hard", lambda x: ref.aggregate_wbg(x, keep_bg=True, hard=True),
                                lambda x: O.aggregate_wbg(x, keep_bg=True, hard=True)),
                               ("wbg_soft", lambda x: ref.aggregate_wbg(x, keep_bg=True), lambda x: O.aggregate_wbg(x, keep_bg=True)),
                               ("sbg", lambda x: ref.aggregate_sbg(x, keep_bg=True), None)):
            r = fn(p)
            if o_fn is not None:
                report[f"agg_K{K}_{mode}_oracle_vs_reference"] = _diff(o_fn(p), r)
            g[f"agg_K{K}_{mode}"] = _np(r)


def clip(ref, fuse, psd, fsd, K, g, report):
    T, h, w, top_k, mem_freq = CLIPS[K]
    net = ref.build_prop(psd, top_k=top_k)
    images, mask, mask2 = clip_inputs(K)
    t0 = time.time()
    core = ref.InferenceCore(net, fuse, images, K, mem_profile=0, mem_freq=mem_freq, device="cpu")
    m1 = core.interact(mask, 0)
    p1 = core.prob.clone()
    m2 = core.interact(mask2, T - 1)
    p2 = core.prob.clone()
    report[f"clip{K}_reference_seconds"] = round(time.time() - t0, 1)
    oc = O.OracleInferenceCore(psd, fsd, images, K, mem_freq=mem_freq, top_k=top_k)
    om1 = oc.interact(mask, 0)
    tr1 = list(oc.bank_trace)
    report[f"clip{K}_prob1_oracle_vs_reference"] = _diff(oc.prob, p1)
    oc.bank_trace = []
    om2 = oc.interact(mask2, T - 1)
    report[f"clip{K}_prob2_oracle_vs_reference"] = _diff(oc.prob, p2)
    report[f"clip{K}_masks_equal"] = [bool((om1 == m1).all()), bool((om2 == m2).all())]
    g[f"clip{K}_masks1"], g[f"clip{K}_masks2"] = m1, m2
    g[f"clip{K}_prob1_sub"] = _np(p1[:, :, 0, ::SUB, ::SUB])
    g[f"clip{K}_prob2_sub"] = _np(p2[:, :, 0, ::SUB, ::SUB])
    g[f"clip{K}_trace1"], g[f"clip{K}_trace2"] = np.array(tr1), np.array(oc.bank_trace)


def main():
    torch.set_grad_enabled(False)
    psd, fsd = Wt.make_prop_state_dict(1234), Wt.make_fusion_state_dict(4321)  # tests/conftest.py
    g, report = {}, {}
    ref = refshim.load_reference()
    try:
        fuse = ref.build_fusion(fsd)
        aggregate(ref, g, report)
        for K in CLIPS:
            clip(ref, fuse, psd, fsd, K, g, report)
    finally:
        ref._restore()
    files = golden_io.save(os.path.join(OUT, "objects.npz"), g)
    report["files"] = [os.path.basename(f) for f in files]
    json.dump(report, open(os.path.join(OUT, "MANIFEST_objects.json"), "w"), indent=1)
    print(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
