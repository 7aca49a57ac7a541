"""Lock-step clips of different object counts against the alternatives a validation run has, in cfg-2 settings
(480p, top-k 20, mem_freq 5, fp16 operands; clips in pinned host memory, mem_profile 2), on one GPU.  8 clips of seeded lengths (20 to 60 frames), seeded
first-interaction frames and seeded object counts (1 to 5):

  (a) the 8 clips in ONE LockstepSession(mixed_objects=True);
  (b) one ragged LockstepSession per object count present (the clips grouped by object count);
  (c) each clip alone through InferenceCore.interact.

Propagated frames and object-frames per second over wall time ended by a device synchronize; the settings alternate
over --runs runs.  Then: (a) against (c) on the timed outputs (bank traces, probabilities, labels); peak device memory
of the first interact of (a) and of (b); and the grouped top-k read (one call for the 8 clips, ragged object counts
and live counts) against one per-set read per object count, at the cfg-2 bank, with CUDA events.

  python tools/mixed_objects_time.py [--runs 3] [--seed 0]

Needs an H100; prints the card and its power limit with the figures."""
from __future__ import annotations

import argparse
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mivos_b200  # noqa: E402
from mivos_b200 import _lib, ops, schedule, synth  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from objects_time import card  # noqa: E402

H, W, TOP_K, MEM_FREQ, C = 480, 854, 20, 5, 8


def make_net(psd):
    net = mivos_b200.PropagationNetwork(top_k=TOP_K, act_dtype=torch.float16)
    net.load_state_dict(psd)
    return net.to("cuda:0")


def make_cores(net, clips, ks):
    # mem_profile 2 (clip in pinned host memory, query features staged 3 frames ahead): the alternating runs keep
    # 3 x 8 clips' result volumes and two networks' workspaces and banks on the device at once; with 105-frame query
    # caches per clip (mem_profile 0 / 1) that does not fit 80 GB at 31 object maps
    return [mivos_b200.InferenceCore(net, None, img, k, mem_freq=MEM_FREQ, mem_profile=2, device="cuda:0")
            for (img, _m), k in zip(clips, ks)]


def timed(fn, cores):
    for c in cores:
        c.reset()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def run_mixed(cores, clips, idxs):
    return timed(lambda: mivos_b200.LockstepSession(cores, mixed_objects=True).interact([m for _i, m in clips], idxs),
                 cores)


def run_by_count(cores, clips, idxs, ks):
    def go():
        for k in sorted(set(ks)):
            sel = [i for i, kk in enumerate(ks) if kk == k]
            mivos_b200.LockstepSession([cores[i] for i in sel], ragged=True).interact(
                [clips[i][1] for i in sel], [idxs[i] for i in sel])
    return timed(go, cores)


def run_solo(cores, clips, idxs):
    def go():
        for c, (_img, m), i in zip(cores, clips, idxs):
            c.interact(m, i)
    return timed(go, cores)


def peak_during(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**20


def read_times(rng, ks, reps=50):
    """The grouped top-k read of the C clips (one call) against one per-set read per object count, cfg-2 bank."""
    dev = torch.device("cuda:0")
    nh, nw = (H + 15) // 16 * 16, (W + 15) // 16 * 16
    hw = (nh // 16) * (nw // 16)
    cap_frames = (schedule.bank_capacity_frames(101, MEM_FREQ, 1, 0) + 15) // 16 * 16
    cap = cap_frames * hw
    N = sum(ks)
    order = sorted(range(C), key=lambda c: ks[c])  # clips of one count adjacent, so a per-set read takes a slice
    kso = [ks[c] for c in order]
    first = [0]
    for k in kso:
        first.append(first[-1] + k)
    g = torch.Generator().manual_seed(1)
    bk = torch.randn((N, cap, 128), generator=g).to(dev)
    bv = torch.randn((N, cap, 512), generator=g).to(dev)
    qk = torch.randn((C, hw, 128), generator=g).to(dev)
    frames = [int(f) for f in rng.integers(1, 22, C)]
    counts = torch.tensor([f * hw for f in frames], dtype=torch.int32, device=dev)
    first_t = torch.tensor(first, dtype=torch.int32, device=dev)
    out = torch.empty((N, hw, 512), device=dev)
    ws = torch.empty(ops.memory_read_workspace_bytes(N, cap, hw, TOP_K), dtype=torch.uint8, device=dev)
    runs = []  # per object count: (map slice, clip slice)
    p = 0
    while p < C:
        q = p
        while q < C and kso[q] == kso[p]:
            q += 1
        runs.append((slice(first[p], first[q]), slice(p, q)))
        p = q

    def grouped():
        ops.memory_read_groups(bk, bv, cap, qk, TOP_K, out, counts, first_t, workspace=ws)

    def per_count():
        for ms, cs in runs:
            ops.memory_read_sets(bk[ms], bv[ms], cap, qk[cs], TOP_K, out[ms], counts[cs], workspace=ws)

    res, ref = {}, None
    for fn in (grouped, per_count):
        fn()
    torch.cuda.synchronize()
    for rnd in range(2):  # alternate, keep the best round of each
        for name, fn in (("grouped", grouped), ("per-count", per_count)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            torch.cuda.synchronize()
            ms = a.elapsed_time(b) / reps
            res[name] = min(res.get(name, ms), ms)
            if ref is None:
                ref = out.clone()
            elif rnd == 1:
                assert torch.equal(out, ref), "grouped and per-count reads differ"
    _lib.poll_kernel_error()
    return kso, frames, hw, len(runs), res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(f"card: {card()}", flush=True)
    rng = np.random.default_rng(args.seed)
    lens = [int(x) for x in rng.integers(20, 61, C)]
    ks = [int(x) for x in rng.integers(1, 6, C)]
    idxs = [int(rng.integers(0, t)) for t in lens]
    clips = [synth.synthetic_clip(t, H, W, k, seed=300 + i) for i, (t, k) in enumerate(zip(lens, ks))]
    print(f"clip lengths {lens}, object counts {ks}, first interactions {idxs}", flush=True)
    psd = synth.make_prop_state_dict()
    # (b) and (c) share one network (their steps live in separate caches of its engine: lock-step and single-clip);
    # (a) has its own, so the alternating runs do not evict each other's steps and graphs
    net_a, net_bc = make_net(psd), make_net(psd)
    nets = {"a": net_a, "b": net_bc, "c": net_bc}
    cores = {s: make_cores(nets[s], clips, ks) for s in "abc"}
    frames = sum(img.shape[1] - 1 for img, _m in clips)  # every frame but the interacted one (both passes)
    obj_frames = sum((img.shape[1] - 1) * k for (img, _m), k in zip(clips, ks))

    peak = {"a": peak_during(lambda: run_mixed(cores["a"], clips, idxs))}
    print(f"peak device memory of the first interact of (a): {peak['a']:.0f} MiB", flush=True)
    peak["b"] = peak_during(lambda: run_by_count(cores["b"], clips, idxs, ks))
    run_solo(cores["c"], clips, idxs)
    print(f"peak device memory of the first interact (steps, banks, workspaces, graphs): mixed (a) {peak['a']:.0f} MiB, "
          f"per object count (b) {peak['b']:.0f} MiB", flush=True)

    times = {"a": [], "b": [], "c": []}
    for r in range(args.runs):
        times["a"].append(run_mixed(cores["a"], clips, idxs))
        times["b"].append(run_by_count(cores["b"], clips, idxs, ks))
        times["c"].append(run_solo(cores["c"], clips, idxs))
        print(f"run {r}: (a) {frames / times['a'][-1]:.1f}  (b) {frames / times['b'][-1]:.1f}  "
              f"(c) {frames / times['c'][-1]:.1f} frames/s", flush=True)
    _lib.poll_kernel_error()
    for key, what in (("a", "one mixed-object session"), ("b", f"{len(set(ks))} ragged sessions, one per object count"),
                      ("c", "one InferenceCore at a time")):
        t = sorted(times[key])
        print(f"({key}) {what}: {frames / t[0]:.1f} frames/s best, {frames / t[len(t) // 2]:.1f} median; "
              f"{obj_frames / t[0]:.1f} object-frames/s best ({frames} frames, {obj_frames} object-frames)", flush=True)

    dmax, dmean, mism, traces = 0.0, 0.0, 0.0, True
    for ca, cc in zip(cores["a"], cores["c"]):
        d = (ca.prob - cc.prob).abs()
        dmax, dmean = max(dmax, float(d.max())), max(dmean, float(d.mean()))
        mism = max(mism, float((ca.masks != cc.masks).float().mean()))
        traces &= ca.bank_trace == cc.bank_trace
    print(f"(a) vs (c): bank traces identical: {traces}; prob max |d| {dmax:.3e}, worst clip mean |d| {dmean:.3e}; "
          f"worst clip label mismatch {mism:.2e}", flush=True)

    del cores, nets, net_a, net_bc
    torch.cuda.empty_cache()
    kso, fr, hw, nruns, res = read_times(rng, ks)
    print(f"top-{TOP_K} read, {C} clips of {kso} objects ({sum(kso)} maps), hw {hw}, live bank frames {fr}: one "
          f"grouped call {res['grouped']:.3f} ms, {nruns} per-set calls (one per object count) "
          f"{res['per-count']:.3f} ms (identical outputs)", flush=True)


if __name__ == "__main__":
    main()
