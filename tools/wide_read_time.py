"""Times the wide top-k memory read (PropagationNetwork(top_k=k) for k > 64, mivos_memory_read_wide) in one process
on one GPU (CUDA events; the card's name and power limit are printed with the numbers):

  * at the bank shapes of cfg-2 (K=1, 20 frames), cfg-3 (K=3, 50 frames) at 480p (hw = 30x54) and cfg-5 (K=5,
    100 frames) at 720p (hw = 45x80), on the same bank: the top-k read at k = 50, the wide read at k = 64, 128, 256
    and 1024, and the dense read;
  * the wide read on a "static camera" bank (one frame's keys repeated in every bank frame with noise of 1e-3: near
    duplicates) at cfg-2 / cfg-3, and on an all-equal-key cfg-2 bank, where every query goes to the exact fallback;
  * `interact()` frames/s of a top_k=128 network at cfg-2 (480p, 1 object, one pass of 20 frames with a bank growing
    to 20 frames), fp16 and TF32.

Usage: python tools/wide_read_time.py [--rounds R] [--out DIR] [--no-sessions]"""
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
from oracle import weights as Wt  # noqa: E402

SHAPES = {"cfg2": (1, 20, 30, 54), "cfg3": (3, 50, 30, 54), "cfg5": (5, 100, 45, 80)}
WIDE_K = (64, 128, 256, 1024)


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


def reads(rounds):
    out = {}
    for name, (K, T, h, w) in SHAPES.items():
        hw, slots = h * w, T * h * w
        g = torch.Generator(device="cuda").manual_seed(1)
        bk = torch.randn((K, slots, 128), generator=g, device="cuda")
        bv = torch.randn((K, slots, 512), generator=g, device="cuda")
        qk = torch.randn((hw, 128), generator=g, device="cuda")
        dst = torch.zeros((K, h + 2, w + 2, 640), device="cuda")
        iters = 3 if name == "cfg5" else 20
        row = {"slots": slots, "hw": hw, "K": K}
        ws = torch.empty(ops.memory_read_workspace_bytes(K, slots, hw, 50), dtype=torch.uint8, device="cuda")
        row["topk_50_ms"] = min(time_op(lambda: ops.memory_read(bk, bv, slots, qk, 50, dst, halo_hw=(h, w),
                                                                workspace=ws), iters) for _ in range(rounds))
        wsw = torch.empty(ops.memory_read_wide_workspace_bytes(K, slots, hw, 1024), dtype=torch.uint8, device="cuda")
        row["wide_workspace_bytes"] = wsw.numel()
        for k in WIDE_K:
            row[f"wide_{k}_ms"] = min(time_op(lambda: ops.memory_read_wide(bk, bv, slots, qk, k, dst, halo_hw=(h, w),
                                                                           workspace=wsw), iters) for _ in range(rounds))
        wsd = torch.empty(ops.memory_read_dense_workspace_bytes(K, slots, hw), dtype=torch.uint8, device="cuda")
        row["dense_ms"] = min(time_op(lambda: ops.memory_read_dense(bk, bv, slots, qk, dst, halo_hw=(h, w),
                                                                    workspace=wsd), iters) for _ in range(rounds))
        out[name] = row
        print(name, json.dumps(row), flush=True)
        del bk, bv, ws, wsw, wsd
        torch.cuda.empty_cache()
    return out


def static_banks(rounds):
    out = {}
    for name in ("cfg2", "cfg3"):
        K, T, h, w = SHAPES[name]
        hw, slots = h * w, T * h * w
        g = torch.Generator(device="cuda").manual_seed(2)
        frame = torch.randn((K, 1, hw, 128), generator=g, device="cuda")
        bk = (frame + 1e-3 * torch.randn((K, T, hw, 128), generator=g, device="cuda")).reshape(K, slots, 128)
        bv = torch.randn((K, slots, 512), generator=g, device="cuda")
        qk = frame[0, 0] + 0.1 * torch.randn((hw, 128), generator=g, device="cuda")
        dst = torch.zeros((K, h + 2, w + 2, 640), device="cuda")
        iters = 3
        wsw = torch.empty(ops.memory_read_wide_workspace_bytes(K, slots, hw, 1024), dtype=torch.uint8, device="cuda")
        row = {}
        for k in (128, 1024):
            row[f"wide_{k}_ms"] = min(time_op(lambda: ops.memory_read_wide(bk, bv, slots, qk, k, dst, halo_hw=(h, w),
                                                                           workspace=wsw), iters) for _ in range(rounds))
        out[name] = row
        print("static", name, json.dumps(row), flush=True)
        if name == "cfg2":
            bk[:] = bk[0, 0]
            out["cfg2_all_equal"] = {f"wide_{k}_ms": time_op(lambda: ops.memory_read_wide(
                bk, bv, slots, qk, k, dst, halo_hw=(h, w), workspace=wsw), 1) for k in (128, 1024)}
            print("all-equal cfg2", json.dumps(out["cfg2_all_equal"]), flush=True)
        del bk, bv, wsw
        torch.cuda.empty_cache()
    return out


def sessions(rounds):
    psd = Wt.make_prop_state_dict(1234)
    images, mask = Wt.synthetic_clip(21, 480, 854, 1, seed=7)
    out = {}
    for act, name in ((torch.float16, "fp16"), (torch.float32, "tf32")):
        net = mivos_b200.PropagationNetwork(top_k=128, act_dtype=act)
        net.load_state_dict(psd, strict=True)
        net = net.cuda()
        best = None
        for _ in range(rounds + 1):  # the first round warms up (graphs, engines)
            core = mivos_b200.InferenceCore(net, None, images, 1, mem_freq=1, device="cuda:0")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            core.interact(mask, 0)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        out[name] = {"frames_per_s": 20 / best}
        print("interact top_k=128", name, json.dumps(out[name]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-sessions", action="store_true")
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    res = {"card": card(), "reads": reads(a.rounds), "static_banks": static_banks(a.rounds)}
    if not a.no_sessions:
        res["interact"] = sessions(a.rounds)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "wide_read_time.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
