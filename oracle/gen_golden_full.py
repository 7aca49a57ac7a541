"""Full-size goldens for every BASELINE.json configuration and for the configuration bench.py times.

TEST INFRASTRUCTURE (see oracle/stm_oracle.py).  Runs the CPU oracle (pinned to the unmodified
reference by oracle/gen_golden.py and tests/test_reference_live.py: max |diff| = 0.0) ONCE per case
on the seeded weights / synthetic clips the GPU tests rebuild from the same seeds, and stores what
the `-m gpu` tests compare against (tests/test_gpu_zzz_fullsize.py):

  masks   u8  [T,h,w]            the oracle's np_masks (full resolution, every frame)
  prob_s  f16 [K+1,T,nh/S,nw/S]  probabilities of every frame on a stride-S pixel grid
  prob_l  f16 [K+1,nh,nw]        probabilities of the LAST propagated frame, full resolution
  trace   i32 [n,2]              (frame, visible bank frames) per propagated frame

Cases (SURVEY.md §8d; BASELINE.json configs[1..4]; clip lengths bounded so the whole file
generates in a few CPU-minutes, per-frame shapes identical to the named configuration):
  cfg2_c{0..3}  480p K=1 top-k 20 mem_freq 5, 101 frames (bank 1 -> 21): the FULL cfg-2 clip, for the
                four clip seeds one bench lane advances in lock-step (bench.py: seed 1234 + c)
  cfg3          480p K=3 top-k 50 mem_freq 5, 27 frames (bank 1 -> 6 + temporary slot)
  cfg4          480p K=2 top-k 50 mem_freq 5, 14 frames, interactions at 0 then 13: 12 frames fused
                by FusionNet (inference_core.py:190-217)
  cfg5          720p K=5 top-k 50 mem_freq 5, 7 frames (45x80 feature maps, no padding)

Run in the build container:  python -m oracle.gen_golden_full [case ...]
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

from oracle import golden_io, stm_oracle as O, weights as Wt  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

# name -> (T, H, W, K, top_k, mem_freq, clip seed, interactions [(frame, mask seed)], stride S)
CASES = {
    "cfg2_c0": (101, 480, 854, 1, 20, 5, 1234, [(0, None)], 16),
    "cfg2_c1": (101, 480, 854, 1, 20, 5, 1235, [(0, None)], 16),
    "cfg2_c2": (101, 480, 854, 1, 20, 5, 1236, [(0, None)], 16),
    "cfg2_c3": (101, 480, 854, 1, 20, 5, 1237, [(0, None)], 16),
    "cfg3": (27, 480, 854, 3, 50, 5, 1234, [(0, None)], 8),
    "cfg4": (14, 480, 854, 2, 50, 5, 1234, [(0, None), (13, 77)], 8),
    "cfg5": (7, 720, 1280, 5, 50, 5, 1234, [(0, None)], 8),
}


def second_mask(k: int, h: int, w: int, seed: int) -> torch.Tensor:
    """A DIFFERENT one-hot mask for the second interaction (cfg-4): the rectangles of
    synthetic_clip shifted by a seeded offset, so the difference masks of fuse_one_frame
    (inference_core.py:233-235) are non-trivial."""
    g = torch.Generator().manual_seed(seed)
    dy, dx = int(torch.randint(10, 40, (1,), generator=g)), int(torch.randint(10, 60, (1,), generator=g))
    mask = torch.zeros((k + 1, 1, h, w))
    for j in range(k):
        y0 = int(h * (0.15 + 0.6 * j / max(k, 1))) + dy
        x0 = int(w * (0.1 + 0.7 * j / max(k, 1))) + dx
        mask[j + 1, 0, y0:y0 + h // 4, x0:x0 + w // 5] = 1
    mask[0] = 1 - mask[1:].sum(0).clamp(0, 1)
    return mask


def build_case(name: str):
    """(images, [(idx, mask)], K, top_k, mem_freq, S) — shared by the generator and the GPU tests."""
    T, H, W, K, top_k, mem_freq, seed, inter, S = CASES[name]
    images, mask0 = Wt.synthetic_clip(T, H, W, K, seed=seed)
    masks = [(idx, mask0 if ms is None else second_mask(K, H, W, ms)) for idx, ms in inter]
    return images, masks, K, top_k, mem_freq, S


def run_case(name: str, psd, fsd) -> dict:
    images, inter, K, top_k, mem_freq, S = build_case(name)
    core = O.OracleInferenceCore(psd, fsd, images, K, mem_freq=mem_freq, top_k=top_k)
    t0 = time.perf_counter()
    out = None
    for idx, m in inter:
        out = core.interact(m, idx)
    dt = time.perf_counter() - t0
    last_ti = core.bank_trace[-1][0]
    golden_io.save(
        os.path.join(OUT, f"full_{name}.npz"),
        dict(masks=out.astype(np.uint8),
             prob_s=core.prob[:, :, 0, ::S, ::S].numpy().astype(np.float16),
             prob_l=core.prob[:, last_ti, 0].numpy().astype(np.float16),
             last_ti=np.int32(last_ti),
             trace=np.asarray(core.bank_trace, dtype=np.int32),
             stride=np.int32(S)))
    frames = len(core.bank_trace)
    return {"frames_propagated": frames, "cpu_seconds": round(dt, 1), "cpu_fps": round(frames / dt, 3),
            "threads": torch.get_num_threads(), "mask_pixels_fg": int((out > 0).sum()),
            "bytes": os.path.getsize(os.path.join(OUT, f"full_{name}.npz"))}


def main(argv):
    torch.set_grad_enabled(False)
    psd = Wt.make_prop_state_dict(1234)
    fsd = Wt.make_fusion_state_dict(4321)
    names = argv or list(CASES)
    man_path = os.path.join(OUT, "MANIFEST_full.json")
    man = json.load(open(man_path)) if os.path.exists(man_path) else {}
    man["torch"] = torch.__version__
    for n in names:
        print(f"[gen_golden_full] {n} ...", flush=True)
        man[n] = run_case(n, psd, fsd)
        print(f"[gen_golden_full] {n}: {man[n]}", flush=True)
        json.dump(man, open(man_path, "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main(sys.argv[1:])
