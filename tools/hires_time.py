"""Times the paths that run above 720p, in one process on one GPU (CUDA events; the card's name and power limit are
printed with the numbers):

  * `interact` frames/s at 1080p (1080x1920, K=2, top-k 50; the clip of tests/test_gpu_zzz_hires.py) for one session,
    fp16 and TF32: the first interaction propagates frames 1..5; the second, at frame 5, propagates AND fuses frames
    4..1, so (its time / 4) - (the first's time / 5) is the cost a fused frame adds;
  * the resident and the streamed attention map at hw = 6912 (64x108), alternated in the same process;
  * the streamed attention map at hw = 8160 (1080p) and 32400 (4K).

Usage: python tools/hires_time.py [--rounds R] [--out DIR]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mivos_b200  # noqa: E402
from mivos_b200 import ops  # noqa: E402
from oracle import gen_golden_hires as GH, weights as Wt  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def time_op(fn, iters):
    """Mean ms per call over `iters` calls (after one warm-up call)."""
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def attention_inputs(h16, w16, seed):
    g = torch.Generator().manual_seed(seed)
    hw = h16 * w16
    mk, qk = (torch.randn(hw, 128, generator=g).cuda() for _ in range(2))
    pos, neg = (torch.rand(1, 1, 16 * h16, 16 * w16, generator=g).cuda() for _ in range(2))
    return mk, qk, h16, w16, pos, neg


def kernels(rounds):
    out = {}
    a = attention_inputs(64, 108, 1)
    res, st = [], []
    for _ in range(rounds):  # alternated: the two paths see the same clocks and neighbours
        res.append(time_op(lambda: ops.attention_map(*a), 20))
        st.append(time_op(lambda: ops.attention_map_streamed(*a), 20))
    out["attention_6912_resident_ms"] = sorted(res)[len(res) // 2]
    out["attention_6912_streamed_ms"] = sorted(st)[len(st) // 2]
    out["attention_6912_spread_ms"] = {"resident": [min(res), max(res)], "streamed": [min(st), max(st)]}
    for name, (h16, w16) in (("8160", (68, 120)), ("32400", (135, 240))):
        b = attention_inputs(h16, w16, 2)
        ms = sorted(time_op(lambda: ops.attention_map_streamed(*b), 10 if h16 < 100 else 3) for _ in range(rounds))
        out[f"attention_{name}_streamed_ms"] = ms[len(ms) // 2]
        hw = h16 * w16
        out[f"attention_{name}_streamed_tflops"] = round(2 * 128 * hw * hw / (ms[len(ms) // 2] * 1e-3) / 1e12, 2)
    return out


def sessions(rounds):
    out = {}
    images, inter, K, top_k, mem_freq, _ = GH.build_clip()
    for act, dt in (("fp16", torch.float16), ("tf32", torch.float32)):
        net = mivos_b200.PropagationNetwork(top_k=top_k, act_dtype=dt)
        net.load_state_dict(Wt.make_prop_state_dict(1234), strict=True)
        net = net.cuda()
        fuse = mivos_b200.FusionNet()
        fuse.load_state_dict(Wt.make_fusion_state_dict(4321), strict=True)
        fuse = fuse.cuda()
        t1s, t2s = [], []
        for r in range(rounds + 1):  # round 0 warms up (graph capture, workspaces)
            core = mivos_b200.InferenceCore(net, fuse, images, K, mem_freq=mem_freq, device="cuda:0")
            ts = []
            for idx, m in inter:
                m = m.cuda()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                core.interact(m, idx)
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            if r:
                t1s.append(ts[0])
                t2s.append(ts[1])
        t1, t2 = sorted(t1s)[len(t1s) // 2], sorted(t2s)[len(t2s) // 2]
        out[f"interact_1080p_{act}_fps"] = round(5 / t1, 2)
        out[f"interact_1080p_{act}_fused_pass_fps"] = round(4 / t2, 2)
        out[f"fused_frame_extra_ms_{act}"] = round((t2 / 4 - t1 / 5) * 1e3, 1)
        del net, fuse, core
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    res = {"card": card()}
    res.update(kernels(a.rounds))
    res.update(sessions(max(1, a.rounds // 2)))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "hires_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
