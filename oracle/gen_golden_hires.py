"""Goldens at 1080p: the frame size DAVIS ships at full resolution and interactive_gui.py --resolution -1 passes.

TEST INFRASTRUCTURE (see oracle/stm_oracle.py).  Runs the CPU oracle (pinned to the unmodified reference by
oracle/gen_golden.py, oracle/gen_golden_s2m.py and tests/test_reference_live.py) ONCE per case on seeded weights
and inputs the GPU test (tests/test_gpu_zzz_hires.py) rebuilds from the same seeds:

  hires_1080p  1080x1920 (padded to 1088x1920: 68x120 = 8160 key pixels), K=2, top-k 50, mem_freq 5, 6 frames,
               interactions at frame 0 and at frame 5: frames 1..4 of the second interaction are fused by
               FusionNet with the attention map at hw = 8160 (above the resident attention kernel's 6912).
               Same arrays as oracle/gen_golden_full.py (masks, prob_s on a stride-8 grid, trace; prob_l
               stored as [(K+1)*nh, nw]).
  s2m_1080p    S2MController.interact (interact/s2m_controller.py:22-37) on a padded 1088x1920 frame with K=2
               objects: 1920 px is wider than the untiled 6-channel stem takes in fp32 (1376) and in fp16 (2760).
               prob_s: the [K,1,nh,nw] result on a stride-4 grid, prob_l: object 1's plane at full resolution.

Run in the build container:  python -m oracle.gen_golden_hires [case ...]
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

from oracle import gen_golden_full as GF, golden_io, s2m_oracle as S, stm_oracle as O, weights as Wt  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
H, W = 1080, 1920
# (T, K, top_k, mem_freq, clip seed, interactions [(frame, mask seed)], stride S)
CLIP = (6, 2, 50, 5, 1080, [(0, None), (5, 77)], 8)
S2M_STRIDE = 4


def build_clip():
    """(images, [(idx, mask)], K, top_k, mem_freq, S): shared by the generator and the GPU test."""
    T, K, top_k, mem_freq, seed, inter, stride = CLIP
    images, mask0 = Wt.synthetic_clip(T, H, W, K, seed=seed)
    masks = [(idx, mask0 if ms is None else GF.second_mask(K, H, W, ms)) for idx, ms in inter]
    return images, masks, K, top_k, mem_freq, stride


def build_s2m(k: int = 2, seed: int = 1081):
    """(padded image [1,3,nh,nw], previous label map [1,nh,nw], scribble labels u8 [H,W], K) as InferenceCore hands
    them to the controller (interactive_gui.py:836-838): 255 = no stroke, 0 = background stroke."""
    g = torch.Generator().manual_seed(seed)
    nh, nw = (H + 15) // 16 * 16, (W + 15) // 16 * 16
    image = torch.randn((1, 3, nh, nw), generator=g)
    prev = torch.zeros((1, nh, nw), dtype=torch.int64)
    prev[:, nh // 5:nh // 2, nw // 6:nw // 2] = 1
    prev[:, nh // 2:3 * nh // 4, nw // 2:5 * nw // 6] = 2
    scr = np.full((H, W), 255, dtype=np.uint8)
    scr[H // 3:H // 3 + 4, W // 5:W // 2] = 1
    scr[2 * H // 3:2 * H // 3 + 4, W // 2:4 * W // 5] = 2
    scr[8:12, 8:W // 3] = 0
    return image, prev, scr, k


def run_clip(psd, fsd) -> dict:
    images, inter, K, top_k, mem_freq, stride = build_clip()
    core = O.OracleInferenceCore(psd, fsd, images, K, mem_freq=mem_freq, top_k=top_k)
    t0 = time.perf_counter()
    out = None
    for idx, m in inter:
        out = core.interact(m, idx)
    last_ti = core.bank_trace[-1][0]
    path = os.path.join(OUT, "hires_1080p.npz")
    files = golden_io.save(path, dict(masks=out.astype(np.uint8),
                                      prob_s=core.prob[:, :, 0, ::stride, ::stride].numpy().astype(np.float16),
                                      # rows of all K+1 planes, so that golden_io can cut it into parts under 1 MB
                                      prob_l=core.prob[:, last_ti, 0].numpy().astype(np.float16).reshape(-1, core.prob.shape[-1]),
                                      last_ti=np.int32(last_ti), trace=np.asarray(core.bank_trace, dtype=np.int32),
                                      stride=np.int32(stride)))
    return {"frames_propagated": len(core.bank_trace), "cpu_seconds": round(time.perf_counter() - t0, 1),
            "files": len(files), "bytes": sum(os.path.getsize(f) for f in files)}


def run_s2m() -> dict:
    sd = Wt.make_s2m_state_dict()
    image, prev, scr, k = build_s2m()
    t0 = time.perf_counter()
    m = S.s2m_controller_interact(sd, image, prev, scr, k)
    path = os.path.join(OUT, "s2m_1080p.npz")
    files = golden_io.save(path, dict(prob_s=m[:, :, ::S2M_STRIDE, ::S2M_STRIDE].numpy().astype(np.float32),
                                      prob_l=m[0, 0].numpy().astype(np.float16), stride=np.int32(S2M_STRIDE)))
    return {"cpu_seconds": round(time.perf_counter() - t0, 1), "files": len(files),
            "bytes": sum(os.path.getsize(f) for f in files)}


def main(argv):
    torch.set_grad_enabled(False)
    names = argv or ["hires_1080p", "s2m_1080p"]
    man_path = os.path.join(OUT, "MANIFEST_hires.json")
    man = json.load(open(man_path)) if os.path.exists(man_path) else {}
    man["torch"] = torch.__version__
    for n in names:
        print(f"[gen_golden_hires] {n} ...", flush=True)
        if n == "hires_1080p":
            man[n] = run_clip(Wt.make_prop_state_dict(1234), Wt.make_fusion_state_dict(4321))
        elif n == "s2m_1080p":
            man[n] = run_s2m()
        else:
            raise SystemExit(f"unknown case {n}")
        print(f"[gen_golden_hires] {n}: {man[n]}", flush=True)
        json.dump(man, open(man_path, "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main(sys.argv[1:])
