"""Lock-step clips with their own pass plans against the same clips one at a time, in cfg-2 settings (480p, 1 object,
top-k 20, mem_freq 5, fp16 operands), on one GPU:

  (a) 8 clips of seeded lengths (25 to 104 frames) and seeded first-interaction frames in ONE LockstepSession
      (ragged: every clip executes its own pass plan);
  (b) the same 8 clips one at a time through InferenceCore.interact;
  (c) 8 clips of one length (the mean of (a)) and one interaction frame through the same-plan session: the ceiling.

Propagated frames per second over wall time ended by a device synchronize; the three settings alternate over --runs
runs.  Then: (a) against (b) on the timed outputs (bank traces, probabilities, labels); peak device memory of the
first session of (a) and of (c); and the per-set top-k read (one call for the 8 clips, ragged counts) against 8
per-clip reads at the cfg-2 bank, with CUDA events.

  python tools/ragged_lockstep_time.py [--runs 3] [--seed 0]

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

H, W, K, TOP_K, MEM_FREQ, C = 480, 854, 1, 20, 5, 8


def make_net(psd):
    net = mivos_b200.PropagationNetwork(top_k=TOP_K, act_dtype=torch.float16)
    net.load_state_dict(psd)
    return net.to("cuda:0")


def make_cores(net, clips):
    return [mivos_b200.InferenceCore(net, None, img, K, mem_freq=MEM_FREQ, device="cuda:0") for img, _m in clips]


def propagated(clips, idxs):
    return sum(img.shape[1] - 1 for img, _m in clips)  # every frame but the interacted one (both passes)


def run_session(cores, clips, idxs, ragged):
    for c in cores:
        c.reset()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mivos_b200.LockstepSession(cores, ragged=ragged).interact([m for _i, m in clips], idxs if ragged else idxs[0])
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def run_solo(cores, clips, idxs):
    for c in cores:
        c.reset()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for c, (_img, m), i in zip(cores, clips, idxs):
        c.interact(m, i)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def peak_during(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**20


def step_memory(net):
    """MiB of the lock-step steps' banks and of the per-frame workspaces of `net`, and the captured graphs."""
    eng = net.engine()
    steps = list(eng.__dict__.get("_lock_steps", {}).values())
    banks = sum(s.bank_k.numel() * 4 + s.bank_v.numel() * 4 for s in steps) / 2**20
    ws = sum(w.bytes() for w in eng._ws_lanes.values()) / 2**20
    return f"{len(steps)} step(s), banks {banks:.0f} MiB, workspaces {ws:.0f} MiB, {sum(len(s.graphs) for s in steps)} graphs"


def read_times(rng, reps=50):
    """The per-set top-k read of C clips (one call) against C per-clip scalar reads, cfg-2 bank, ragged counts."""
    dev = torch.device("cuda:0")
    nh, nw = (H + 15) // 16 * 16, (W + 15) // 16 * 16
    hw = (nh // 16) * (nw // 16)
    cap_frames = (schedule.bank_capacity_frames(101, MEM_FREQ, 1, 0) + 15) // 16 * 16
    cap = cap_frames * hw
    g = torch.Generator().manual_seed(1)
    bk = torch.randn((C * K, cap, 128), generator=g).to(dev)
    bv = torch.randn((C * K, cap, 512), generator=g).to(dev)
    qk = torch.randn((C, hw, 128), generator=g).to(dev)
    frames = [int(f) for f in rng.integers(1, 22, C)]
    counts = torch.tensor([f * hw for f in frames], dtype=torch.int32, device=dev)
    out = torch.empty((C * K, hw, 512), device=dev)
    ws_sets = torch.empty(ops.memory_read_workspace_bytes(C * K, cap, hw, TOP_K), dtype=torch.uint8, device=dev)
    ws_one = torch.empty(ops.memory_read_workspace_bytes(K, cap, hw, TOP_K), dtype=torch.uint8, device=dev)
    dyn = [counts[c:c + 1] for c in range(C)]

    def per_set():
        ops.memory_read_sets(bk, bv, cap, qk, TOP_K, out, counts, workspace=ws_sets)

    def per_clip():
        for c in range(C):
            ops.memory_read(bk[c * K:(c + 1) * K], bv[c * K:(c + 1) * K], cap, qk[c], TOP_K, out[c * K:(c + 1) * K],
                            workspace=ws_one, dyn_slots=dyn[c])

    res = {}
    for name, fn in (("per-set", per_set), ("per-clip", per_clip)):
        fn()
        torch.cuda.synchronize()
    ref = None
    for rnd in range(2):  # alternate, keep the best round of each
        for name, fn in (("per-set", per_set), ("per-clip", per_clip)):
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
                assert torch.equal(out, ref), "per-set and per-clip reads differ"
    _lib.poll_kernel_error()
    return frames, hw, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(f"card: {card()}", flush=True)
    rng = np.random.default_rng(args.seed)
    lens = [int(x) for x in rng.integers(25, 105, C)]
    idxs = [int(rng.integers(0, t)) for t in lens]
    clips = [synth.synthetic_clip(t, H, W, K, seed=100 + i) for i, t in enumerate(lens)]
    L = int(round(np.mean(lens)))
    i_eq = int(rng.integers(0, L))
    clips_eq = [synth.synthetic_clip(L, H, W, K, seed=200 + i) for i in range(C)]
    print(f"(a)/(b) clip lengths {lens}, first interactions {idxs}; (c) {C} clips of {L} frames, interaction {i_eq}",
          flush=True)
    psd = synth.make_prop_state_dict()
    net_a, net_b, net_c = make_net(psd), make_net(psd), make_net(psd)
    cores_a, cores_b, cores_c = make_cores(net_a, clips), make_cores(net_b, clips), make_cores(net_c, clips_eq)
    n_ab, n_c = propagated(clips, idxs), propagated(clips_eq, [i_eq] * C)

    # warm-up (workspaces, graph capture), peak memory of the first session of (a) and (c) on fresh networks
    peak_a = peak_during(lambda: run_session(cores_a, clips, idxs, True))
    peak_c = peak_during(lambda: run_session(cores_c, clips_eq, [i_eq] * C, False))
    run_solo(cores_b, clips, idxs)
    print(f"peak device memory of a session's first interact (steps, banks, workspaces, graphs): ragged (a) "
          f"{peak_a:.0f} MiB, same-plan (c) {peak_c:.0f} MiB", flush=True)
    print(f"  (a) {step_memory(net_a)}; (c) {step_memory(net_c)}", flush=True)

    times = {"a": [], "b": [], "c": []}
    for r in range(args.runs):
        times["a"].append(run_session(cores_a, clips, idxs, True))
        times["b"].append(run_solo(cores_b, clips, idxs))
        times["c"].append(run_session(cores_c, clips_eq, [i_eq] * C, False))
        print(f"run {r}: (a) {n_ab / times['a'][-1]:.1f}  (b) {n_ab / times['b'][-1]:.1f}  "
              f"(c) {n_c / times['c'][-1]:.1f} frames/s", flush=True)
    _lib.poll_kernel_error()
    for key, n, what in (("a", n_ab, "ragged lock-step session"), ("b", n_ab, "one InferenceCore at a time"),
                         ("c", n_c, "same-plan session, equal clips")):
        fps = sorted(n / t for t in times[key])
        print(f"({key}) {what}: {fps[-1]:.1f} frames/s best, {fps[len(fps) // 2]:.1f} median "
              f"({n} propagated frames)", flush=True)

    # (a) against (b) on the outputs of the last timed run
    dmax, dmean, mism, traces = 0.0, 0.0, 0.0, True
    for ca, cb in zip(cores_a, cores_b):
        d = (ca.prob - cb.prob).abs()
        dmax, dmean = max(dmax, float(d.max())), max(dmean, float(d.mean()))
        mism = max(mism, float((ca.masks != cb.masks).float().mean()))
        traces &= ca.bank_trace == cb.bank_trace
    print(f"(a) vs (b): bank traces identical: {traces}; prob max |d| {dmax:.3e}, worst clip mean |d| {dmean:.3e}; "
          f"worst clip label mismatch {mism:.2e}", flush=True)

    del cores_a, cores_b, cores_c, net_a, net_b, net_c
    torch.cuda.empty_cache()
    frames, hw, res = read_times(rng)
    print(f"top-{TOP_K} read, {C} clips x {K} object, hw {hw}, live bank frames {frames}: one per-set call "
          f"{res['per-set']:.3f} ms, {C} per-clip calls {res['per-clip']:.3f} ms (identical outputs)", flush=True)


if __name__ == "__main__":
    main()
