"""Times the dense memory read (PropagationNetwork(top_k=None), mivos_memory_read_dense) in one process on one GPU
(CUDA events; the card's name and power limit are printed with the numbers):

  * at the bank shapes of cfg-2 (K=1, 20 frames), cfg-3 (K=3, 50 frames) at 480p (hw = 30x54) and cfg-5 (K=5,
    100 frames) at 720p (hw = 45x80), on the same bank:
      - the dense read, with algorithmic TFLOP/s 2*(128+512)*slots*hw*K (3xTF32 counted once) and the share of the
        495 TFLOP/s dense TF32 data-sheet peak of the H100 SXM;
      - the top-k read at top_k 20 and 50;
      - what the reference runs: PyTorch eager bmm -> softmax(dim=1) -> bmm in fp32 with TF32 off, per object;
  * `interact()` frames/s of a top_k=None network at cfg-2 (480p, 1 object, one pass of 20 frames with a bank
    growing to 20 frames), fp16 and TF32, next to the top_k=20 network on the same clip.

Usage: python tools/dense_read_time.py [--rounds R] [--out DIR] [--no-sessions]"""
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

PEAK_TF32 = 495e12
SHAPES = {"cfg2": (1, 20, 30, 54), "cfg3": (3, 50, 30, 54), "cfg5": (5, 100, 45, 80)}


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


def median(xs):
    return sorted(xs)[len(xs) // 2]


def reads(rounds):
    out = {}
    for name, (K, T, h, w) in SHAPES.items():
        hw, n = h * w, T * h * w
        g = torch.Generator(device="cuda").manual_seed(1)
        bk = torch.randn((K, n, 128), generator=g, device="cuda")
        bv = torch.randn((K, n, 512), generator=g, device="cuda")
        qk = torch.randn((hw, 128), generator=g, device="cuda")
        cat = ops.halo_zeros(K, h, w, 1024, torch.device("cuda"))
        wsd = torch.empty(ops.memory_read_dense_workspace_bytes(K, n, hw), dtype=torch.uint8, device="cuda")
        wst = torch.empty(ops.memory_read_workspace_bytes(K, n, hw, 50), dtype=torch.uint8, device="cuda")
        iters = 20 if K * n * hw < 3e9 else 5
        dense = median([time_op(lambda: ops.memory_read_dense(bk, bv, n, qk, cat, halo_hw=(h, w), workspace=wsd), iters)
                        for _ in range(rounds)])
        row = {"dense_ms": round(dense, 3), "workspace_mb": round(wsd.numel() / 2 ** 20, 1)}
        flops = 2 * (128 + 512) * n * hw * K
        row["dense_tflops"] = round(flops / (dense * 1e-3) / 1e12, 1)
        row["dense_share_of_tf32_peak"] = round(flops / (dense * 1e-3) / PEAK_TF32, 3)
        for k in (20, 50):
            row[f"top{k}_ms"] = round(median([time_op(lambda: ops.memory_read(bk, bv, n, qk, k, cat, halo_hw=(h, w),
                                                                               workspace=wst), iters)
                                              for _ in range(rounds)]), 3)
        mk = bk.transpose(1, 2)  # [K, 128, slots]: the reference's layout of the bank (a view)
        mv = bv.transpose(1, 2)
        q = (qk.t() / 128 ** 0.5).contiguous()

        def eager():
            for o in range(K):  # the reference's bmm over B = K objects, one object at a time (same flops)
                aff = torch.softmax(torch.mm(mk[o].t(), q), dim=0)   # [slots, hw]
                torch.mm(mv[o], aff)
        prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            row["eager_fp32_ms"] = round(median([time_op(eager, max(2, iters // 4)) for _ in range(max(1, rounds // 2))]), 3)
            # where the eager time goes, object 0: the two GEMMs and the softmax over the memory axis
            aff = torch.mm(mk[0].t(), q)
            row["eager_obj0_ms"] = {"qk_mm": round(time_op(lambda: torch.mm(mk[0].t(), q), 3), 3),
                                    "softmax": round(time_op(lambda: torch.softmax(aff, dim=0), 3), 3),
                                    "pv_mm": round(time_op(lambda: torch.mm(mv[0], aff), 3), 3)}
            del aff
        finally:
            torch.backends.cuda.matmul.allow_tf32 = prev
        row["speedup_vs_eager"] = round(row["eager_fp32_ms"] / dense, 2)
        out[name] = row
        del bk, bv, qk, cat, wsd, wst
        torch.cuda.empty_cache()
    return out


def sessions(rounds):
    out = {}
    images, mask = Wt.synthetic_clip(21, 480, 854, 1, seed=3)
    for label, top_k in (("dense", None), ("top20", 20)):
        for act, dt in (("fp16", torch.float16), ("tf32", torch.float32)):
            net = mivos_b200.PropagationNetwork(top_k=top_k, act_dtype=dt)
            net.load_state_dict(Wt.make_prop_state_dict(1234), strict=True)
            net = net.cuda()
            ts = []
            for r in range(rounds + 1):  # round 0 warms up (graph capture, workspaces)
                core = mivos_b200.InferenceCore(net, None, images, 1, mem_freq=1, device="cuda:0")
                m = mask.cuda()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                core.interact(m, 0)
                torch.cuda.synchronize()
                if r:
                    ts.append(time.perf_counter() - t0)
            out[f"interact_cfg2_{label}_{act}_fps"] = round(20 / median(ts), 2)
            del net, core
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-sessions", action="store_true")
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    res = {"card": card()}
    res["reads"] = reads(a.rounds)
    if not a.no_sessions:
        res.update(sessions(max(1, a.rounds // 2)))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "dense_read_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
