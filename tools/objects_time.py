"""Per-frame time of InferenceCore.interact at 480p for K in {16, 17, 32, 64} objects (16: one object chunk, above:
ceil(K / 16) chunks), in fp16 and TF32, and the time of the memorize stem gather at K = 255 (its "others" channel
is a sum over all K masks for each of the K objects: O(K^2) per pixel).

  python tools/objects_time.py [--frames T] [--reps R]

Needs an H100; prints the card and its power limit with the figures."""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mivos_b200  # noqa: E402
from mivos_b200 import _lib, ops, synth  # noqa: E402
from mivos_b200.engine import object_chunks  # noqa: E402


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name() + ", power limit unknown"
    return q


def interact_ms_per_frame(net, images, mask, K, reps):
    core = mivos_b200.InferenceCore(net, None, images, K, mem_freq=5, device="cuda:0")
    core.interact(mask, 0)  # warm-up: workspaces, graph capture
    T = images.shape[1]
    times = []
    for _ in range(reps):
        core.reset()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        core.interact(mask, 0)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) / (T - 1))  # T - 1 propagated frames (interaction on frame 0)
    _lib.poll_kernel_error()
    return min(times), sorted(times)[len(times) // 2]


def stem_ms(K, H, W, f16, reps):
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    frame = torch.randn((1, 3, H, W), generator=g).to(dev)
    masks = torch.rand((K, 1, H, W), generator=g).to(dev)
    rows = (H // 2 + 2) * (W // 2 + 2)
    n_max = max(n for _, n in object_chunks(K))
    out = torch.empty((n_max * rows, 128 if f16 else 96), dtype=torch.float16 if f16 else torch.float32, device=dev)
    for k0, n in object_chunks(K):
        ops.stem_gather_range(frame, masks, k0, n, out)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        for k0, n in object_chunks(K):
            ops.stem_gather_range(frame, masks, k0, n, out)
    b.record()
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(f"card: {card()}")
    psd = synth.make_prop_state_dict()
    H, W = 480, 854
    for act, name in ((torch.float16, "fp16"), (torch.float32, "tf32")):
        net = mivos_b200.PropagationNetwork(top_k=50, act_dtype=act)
        net.load_state_dict(psd)
        net = net.to("cuda:0")
        for K in (16, 17, 32, 64):
            images, mask = synth.synthetic_clip(args.frames, H, W, K, seed=K)
            best, med = interact_ms_per_frame(net, images, mask, K, args.reps)
            print(f"interact 480p {name} K={K:3d} chunks={len(object_chunks(K))}: {best:8.2f} ms/frame (median {med:.2f}, "
                  f"{best / K:.3f} ms per object-frame)", flush=True)
        del net
        torch.cuda.empty_cache()
    for f16 in (True, False):
        ms = stem_ms(255, 480, 864, f16, args.reps * 3)
        print(f"stem gather 480p K=255 ({len(object_chunks(255))} chunks, {'fp16' if f16 else 'fp32'} matrix): "
              f"{ms:.2f} ms per memorize", flush=True)


if __name__ == "__main__":
    main()
