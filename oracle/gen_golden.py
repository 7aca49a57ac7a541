"""Generate tests/golden/*.npz by running the UNMODIFIED reference (imported from /root/reference
through oracle/refshim.py) on seeded weights and inputs, and check the oracle restatement against
it on the spot.  Run in the build container:  python -m oracle.gen_golden

TEST INFRASTRUCTURE (see oracle/stm_oracle.py).  The fixtures pin the oracle: tests replay them
without the reference being present (the GPU box has no /root/reference).
"""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import golden_io, refshim, stm_oracle as O, weights as Wt  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def _np(t):
    return t.detach().cpu().numpy()


def _cmp(name, a, b, report):
    d = float((a.double() - b.double()).abs().max())
    s = float(b.double().abs().max())
    report[name] = {"max_abs_diff_oracle_vs_reference": d, "ref_abs_max": s}
    return d


def main():
    torch.set_grad_enabled(False)
    torch.manual_seed(0)
    os.makedirs(OUT, exist_ok=True)
    ref = refshim.load_reference()
    psd = Wt.make_prop_state_dict(1234)
    fsd = Wt.make_fusion_state_dict(4321)
    report = {"torch": torch.__version__, "prop_keys": len(psd), "fusion_keys": len(fsd)}

    # strict load proves our key/shape table equals the reference's (597 / 12 tensors)
    net20 = ref.build_prop(psd, top_k=20)
    net50 = ref.build_prop(psd, top_k=50)
    fuse = ref.build_fusion(fsd)
    assert len(net20.state_dict()) == len(psd) == 597, len(psd)
    assert len(fuse.state_dict()) == len(fsd) == 12

    # ------------------------------------------------------------------ op-level goldens (low res)
    H, W, K = 96, 128, 2
    images, mask = Wt.synthetic_clip(4, H, W, K, seed=7)
    frame = images[:, 0]
    g = {}
    qv_ref = net20.get_query_values(frame)
    qv_orc = O.get_query_values(psd, frame)
    for n, a, b in zip(("f16", "f8", "f4", "k16", "v16"), qv_orc, qv_ref):
        _cmp("qv_" + n, a, b, report)
    g.update(frame=_np(frame), mask=_np(mask), f16=_np(qv_ref[0]), f8=_np(qv_ref[1][:, ::4]), f4=_np(qv_ref[2][:, ::8]),
             k16=_np(qv_ref[3]), v16=_np(qv_ref[4]))
    mk_ref, mv_ref = net20.memorize(frame, mask[1:])
    mk_orc, mv_orc = O.memorize(psd, frame, mask[1:])
    _cmp("mem_k", mk_orc, mk_ref, report)
    _cmp("mem_v", mv_orc, mv_ref, report)
    g.update(mem_k=_np(mk_ref), mem_v=_np(mv_ref))

    # bank of 3 frames (soft masks so the mask channels are exercised with non-binary values)
    soft = [mask[1:], (mask[1:] * 0.7 + 0.1), torch.rand(K, 1, H, W, generator=torch.Generator().manual_seed(3))]
    ks, vs = zip(*[net20.memorize(images[:, i], soft[i]) for i in range(3)])
    keys, values = torch.cat(ks, 2), torch.cat(vs, 2)
    qv3 = net20.get_query_values(images[:, 3])
    rd_ref = net20.memory(keys[0:1], values[0:1], qv3[3])
    rd_orc = O.memory_read(keys[0:1], values[0:1], qv3[3], 20)
    _cmp("read_top20", rd_orc, rd_ref, report)
    seg_ref = net20.segment_with_query(keys, values, *qv3)
    seg_orc = O.segment_with_query(psd, keys, values, *qv3, top_k=20)
    _cmp("segment", seg_orc, seg_ref, report)
    agg_ref = ref.aggregate_wbg(seg_ref, keep_bg=True)
    _cmp("aggregate", O.aggregate_wbg(seg_orc, keep_bg=True), agg_ref, report)
    g.update(frame3=_np(images[:, 3]), keys=_np(keys), values=_np(values), read=_np(rd_ref), seg=_np(seg_ref),
             agg=_np(agg_ref), qk3=_np(qv3[3]))

    # attention + fusion
    gg = torch.Generator().manual_seed(11)
    pos = torch.rand((1, 1, H, W), generator=gg)
    neg = torch.rand((1, 1, H, W), generator=gg)
    at_ref = net20.get_attention(mk_ref[0:1], pos, neg, qv3[3])
    at_orc = O.get_attention(None, mk_ref[0:1], pos, neg, qv3[3])
    _cmp("attention", at_orc, at_ref, report)
    dist = torch.tensor([[0.25, 0.75]])
    fu_ref = fuse(images[:, 3], seg_ref[0:1], agg_ref[1:2], at_ref, dist)
    fu_orc = O.fusion_net(fsd, images[:, 3], seg_ref[0:1], agg_ref[1:2], at_ref, dist)
    _cmp("fusion", fu_orc, fu_ref, report)
    g.update(pos=_np(pos), neg=_np(neg), attn=_np(at_ref), fuse=_np(fu_ref), dist=_np(dist))
    golden_io.save(os.path.join(OUT, "ops_lowres.npz"), g)

    # ------------------------------------------------------------------ memory-read goldens (random tensors)
    gm = torch.Generator().manual_seed(5)
    mk = torch.randn((2, 128, 4, 6, 8), generator=gm)
    mv = torch.randn((2, 512, 4, 6, 8), generator=gm)
    qk = torch.randn((1, 128, 6, 8), generator=gm)
    rd = {}
    for k_, net in ((20, net20), (50, net50)):
        r = torch.cat([net.memory(mk[i:i + 1], mv[i:i + 1], qk) for i in range(2)], 0)
        o = torch.cat([O.memory_read(mk[i:i + 1], mv[i:i + 1], qk, k_) for i in range(2)], 0)
        _cmp(f"memread_top{k_}", o, r, report)
        rd[f"out{k_}"] = _np(r)
    golden_io.save(os.path.join(OUT, "memread.npz"), dict(mk=_np(mk), mv=_np(mv), qk=_np(qk), **rd))

    # ------------------------------------------------------------------ whole-clip golden, low res, with fusion
    T, h, w, K = 6, 64, 88, 2  # 88 -> padded to 96: exercises pad/unpad
    images, mask = Wt.synthetic_clip(T, h, w, K, seed=21)
    _, mask2 = Wt.synthetic_clip(T, h, w, K, seed=22)
    mask2 = torch.roll(mask2, shifts=(5, 9), dims=(2, 3))
    core = ref.InferenceCore(net20, fuse, images, K, mem_profile=0, mem_freq=2, device="cpu")
    cb = {"total": [], "steps": 0}
    m1 = core.interact(mask, 0, total_cb=lambda n: cb["total"].append(n), step_cb=lambda: cb.__setitem__("steps", cb["steps"] + 1))
    p1 = core.prob.clone()
    m2 = core.interact(mask2, T - 1)
    p2 = core.prob.clone()
    oc = O.OracleInferenceCore(psd, fsd, images, K, mem_freq=2, top_k=20)
    om1 = oc.interact(mask, 0)
    _cmp("clip_prob_after_interact1", oc.prob, p1, report)
    om2 = oc.interact(mask2, T - 1)
    _cmp("clip_prob_after_interact2", oc.prob, p2, report)
    report["clip_masks_equal"] = [bool((om1 == m1).all()), bool((om2 == m2).all())]
    report["clip_callbacks"] = {"total": cb["total"], "steps": cb["steps"]}
    report["clip_bank_trace"] = oc.bank_trace
    np.savez_compressed(os.path.join(OUT, "clip_lowres.npz"), images=_np(images), mask=_np(mask), mask2=_np(mask2),
                        masks1=m1, masks2=m2, prob1=_np(p1), prob2=_np(p2), pad=np.array(core.pad))

    # ------------------------------------------------------------------ BASELINE configs[0]: 480p plumbing
    T, h, w, K = 5, 480, 854, 1
    images, mask = Wt.synthetic_clip(T, h, w, K, seed=1234)
    t0 = time.time()
    core = ref.InferenceCore(net50, None, images, K, mem_profile=0, mem_freq=2, device="cpu")
    m = core.interact(mask, 0)
    report["cfg1_reference_seconds"] = time.time() - t0
    oc = O.OracleInferenceCore(psd, None, images, K, mem_freq=2, top_k=50)
    om = oc.interact(mask, 0)
    _cmp("cfg1_prob", oc.prob, core.prob, report)
    report["cfg1_masks_equal"] = bool((om == m).all())
    report["cfg1_bank_trace"] = oc.bank_trace
    report["cfg1_fg_fraction"] = float((m > 0).mean())
    np.savez_compressed(os.path.join(OUT, "cfg1_480p.npz"), masks=m, prob_sub=_np(core.prob[:, :, :, ::8, ::8]),
                        pad=np.array(core.pad))
    ref._restore()
    json.dump(report, open(os.path.join(OUT, "MANIFEST.json"), "w"), indent=1)
    print(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
