"""Host results (InferenceCore(result_dev="cpu")) against device results, on one GPU, in one call; the two settings
alternate over --runs runs each:

  (1) one cfg-2 interact: 480p (480x854 -> 480x864), 1 object, 101 frames, top-k 20, fp16 operands, mem_profile 0;
  (2) an 8-clip LockstepSession(mixed_objects=True) at mem_profile 2 (seeded lengths 20 to 60, 1 to 5 objects);
  (3) a 1080p clip of 3 objects and a 4K clip of 1 object at mem_profile 2: frames/s and peak device memory;
  (4) a clip whose device results do not fit the card (480p, 255 objects, 101 frames: prob and bank together exceed
      it) with host results, if the host's MemAvailable holds its host volumes and clip; else the reason it is skipped.

Frames per second over wall time ended by a device synchronize.  The bytes that cross PCIe per frame are computed
from the shapes (planes, then the two label maps); the outputs of the two settings are compared bit for bit.

  python tools/host_results_time.py [--runs 3] [--hires-frames 40] [--skip-over]

Needs an H100; prints the card and its power limit with the figures."""
from __future__ import annotations

import argparse
import gc
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mivos_b200  # noqa: E402
from mivos_b200 import schedule, synth  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from objects_time import card  # noqa: E402

SETTINGS = (("device", None), ("host", "cpu"))


def make_net(psd, top_k):
    net = mivos_b200.PropagationNetwork(top_k=top_k, act_dtype=torch.float16)
    net.load_state_dict(psd)
    return net.to("cuda:0")


def pcie_mb(K, H, W):
    nh, nw = (H + 15) // 16 * 16, (W + 15) // 16 * 16
    return (K + 1) * nh * nw * 4 / 1e6, (nh * nw + H * W) / 1e6


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def fmt(name, frames, secs):
    return f"{name} " + " ".join(f"{frames / s:7.1f}" for s in secs) + " frames/s"


def single(psd, runs):
    H, W, K, T = 480, 854, 1, 101
    net = make_net(psd, 20)
    images, mask = synth.synthetic_clip(T, H, W, K, seed=1)
    cores = {n: mivos_b200.InferenceCore(net, None, images, K, mem_freq=5, device="cuda:0", result_dev=r)
             for n, r in SETTINGS}
    for c in cores.values():
        c.interact(mask, 0)  # warm-up: workspaces, graph capture
    secs = {n: [] for n, _ in SETTINGS}
    for _ in range(runs):
        for n, c in cores.items():
            c.reset()
            secs[n].append(timed(lambda: c.interact(mask, 0))[0])
    same = torch.equal(cores["device"].prob.cpu(), cores["host"].prob) and np.array_equal(*(c.np_masks for c in cores.values()))
    p, lab = pcie_mb(K, H, W)
    print(f"(1) cfg-2 interact, {T - 1} propagated frames; PCIe per frame {p:.1f} MB planes + {lab:.1f} MB labels; "
          f"bit-identical: {same}")
    for n, _ in SETTINGS:
        print("    " + fmt(f"{n:6s}", T - 1, secs[n]))


def mixed(psd, runs):
    H, W, C = 480, 854, 8
    rng = np.random.default_rng(0)
    lens = [int(x) for x in rng.integers(20, 61, C)]
    ks = [int(x) for x in rng.integers(1, 6, C)]
    idxs = [int(rng.integers(0, t)) for t in lens]
    clips = [synth.synthetic_clip(t, H, W, k, seed=10 + i) for i, (t, k) in enumerate(zip(lens, ks))]
    net = make_net(psd, 20)
    cores = {n: [mivos_b200.InferenceCore(net, None, img, k, mem_freq=5, mem_profile=2, device="cuda:0", result_dev=r)
                 for (img, _m), k in zip(clips, ks)] for n, r in SETTINGS}
    frames = sum(t - 1 for t in lens)

    def go(cs):
        for c in cs:
            c.reset()
        return timed(lambda: mivos_b200.LockstepSession(cs, mixed_objects=True).interact([m for _i, m in clips], idxs))[0]

    for cs in cores.values():
        go(cs)
    secs = {n: [go(cores[n]) for _ in range(1)] for n, _ in SETTINGS}
    for _ in range(runs - 1):
        for n, _ in SETTINGS:
            secs[n].append(go(cores[n]))
    same = all(torch.equal(a.prob.cpu(), b.prob) for a, b in zip(cores["device"], cores["host"]))
    print(f"(2) 8-clip mixed_objects session, mem_profile 2 (lengths {lens}, objects {ks}), {frames} propagated "
          f"clip-frames; bit-identical: {same}")
    for n, _ in SETTINGS:
        print("    " + fmt(f"{n:6s}", frames, secs[n]))


def hires(psd, runs, T):
    for H, W, K in ((1080, 1920, 3), (2160, 3840, 1)):
        images, mask = synth.synthetic_clip(T, H, W, K, seed=5)
        net = make_net(psd, 50)
        secs, peaks, probs = {n: [] for n, _ in SETTINGS}, {}, {}
        for r in range(runs):
            for n, rd in SETTINGS:
                gc.collect()
                torch.cuda.empty_cache()
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                core = mivos_b200.InferenceCore(net, None, images, K, mem_freq=5, mem_profile=2, device="cuda:0",
                                                result_dev=rd)
                core.interact(mask, 0)  # warm-up (first run: graph capture)
                core.reset()
                secs[n].append(timed(lambda: core.interact(mask, 0))[0])
                peaks[n] = (torch.cuda.max_memory_allocated() - base) / 2**30
                if r == 0:
                    probs[n] = core.prob[:, -1].cpu()
                del core
        p, lab = pcie_mb(K, H, W)
        print(f"(3) {H}x{W}, {K} object(s), {T} frames, mem_profile 2; PCIe per frame {p:.1f} MB planes + {lab:.1f} MB "
              f"labels; bit-identical (last frame): {torch.equal(probs['device'], probs['host'])}")
        for n, _ in SETTINGS:
            print("    " + fmt(f"{n:6s}", T - 1, secs[n]) + f", peak device memory {peaks[n]:.2f} GiB over the network")
        del net
        gc.collect()
        torch.cuda.empty_cache()


def mem_available() -> int:
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def over_capacity(psd):
    H, W, K, T = 480, 854, 255, 101
    nh, nw = 480, 864
    hw = (nh // 16) * (nw // 16)
    cap = (schedule.bank_capacity_frames(T, 5, 1, 0) + 15) // 16 * 16
    bank = K * cap * hw * (128 + 512) * 4
    results = (K + 1) * T * nh * nw * 4 + T * (nh * nw + H * W)
    card_bytes = torch.cuda.get_device_properties(0).total_memory
    host_need = results + T * 3 * nh * nw * 4 * 2 + (4 << 30)  # volumes, the clip (padded copy + pinned), headroom
    print(f"(4) 480p, {K} objects, {T} frames: bank {bank / 1e9:.1f} GB + device results {results / 1e9:.1f} GB = "
          f"{(bank + results) / 1e9:.1f} GB against {card_bytes / 1e9:.1f} GB on the card")
    avail = mem_available()
    if avail < host_need:
        print(f"    skipped: the host has {avail / 1e9:.1f} GB available, the run needs about {host_need / 1e9:.1f} GB")
        return
    images, mask = synth.synthetic_clip(T, H, W, K, seed=7)
    net = make_net(psd, 20)
    torch.cuda.reset_peak_memory_stats()
    try:
        core = mivos_b200.InferenceCore(net, None, images, K, mem_freq=5, mem_profile=2, device="cuda:0",
                                        result_dev="cpu")
        secs, out = timed(lambda: core.interact(mask, 0))
        print(f"    host results: ran, {(T - 1) / secs:.1f} frames/s, peak device memory "
              f"{torch.cuda.max_memory_allocated() / 2**30:.1f} GiB, labels {np.bincount(out.ravel(), minlength=K + 1)[:4]}...")
    except RuntimeError as e:  # MivosError included
        print(f"    host results: failed: {e}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--hires-frames", type=int, default=40)
    ap.add_argument("--skip-over", action="store_true")
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    print(f"card: {card()}")
    psd = synth.make_prop_state_dict()
    single(psd, a.runs)
    mixed(psd, a.runs)
    hires(psd, a.runs, a.hires_frames)
    if not a.skip_over:
        over_capacity(psd)
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
