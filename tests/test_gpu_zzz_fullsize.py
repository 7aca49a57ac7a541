"""GPU: network-level parity at the sizes BASELINE.json names, against the full-size goldens the CPU
oracle produced (oracle/gen_golden_full.py; tests/golden/full_*.npz), on both element types:

  cfg-2  480p, 1 object, top-k 20, the WHOLE 101-frame clip (100 frames of feedback through memorize,
         bank 1 -> 21 frames) — through a single InferenceCore (the call the unchanged reference
         callers make) AND through the configuration bench.py times: its concurrent lanes (own network
         object, CUDA stream and Python thread each) x LockstepSession of 4 clips;
  cfg-3  480p, 3 objects, top-k 50, 27 frames (multi-frame bank + temporary slot);
  cfg-4  480p, 2 objects, two interactions (frame 0 then 13): 12 frames through fuse_one_frame /
         FusionNet / get_attention at full resolution;
  cfg-5  720p, 5 objects, top-k 50 (45x80 feature maps, unpadded, K=5 "others" masks).
  plus mem_profile 2 / 3 (3- and 1-frame query / image caches with wholesale flushes) on the GPU.

What is asserted, per case and element type (reference: inference_core.py:122-271):
  * bank bookkeeping identical to the oracle's trace (bit-exact);
  * u8 masks: fraction of differing pixels, worst frame and LAST frame;
  * probabilities: max |dp| over every frame on the golden's pixel grid, and over the full-resolution
    last frame; mean |dp|.
The drift curve (per-frame mask mismatch and max |dp|) is written to $MIVOS_DRIFT_DIR/drift_*.json when
that variable names a directory (tools/drift_table.py tabulates them).

Stated tolerances (fp16 / TF32 operands vs the fp32 reference; both element types share them):
  P_MAX   max |dp| <= 6e-2 anywhere on any frame (single-frame tests: 3e-2; a 100-frame chain feeds each
          frame's probabilities back through memorize, so the bound is doubled for drift).  Measured on an
          H100 80GB HBM3 at a 400 W power limit (another card than the 700 W one of the benchmark numbers in
          README.md; parity does not depend on it): 0.7-2.9e-2 worst over the single-session clips, with no growth
          along the clip (errors do not accumulate through the memory bank).
  P_MEAN  mean |dp| <= 2e-3 (measured on the same H100: 1.8e-5 .. 1.7e-4)
  MASKS   (i) every DECIDED pixel agrees exactly: wherever the oracle's best label leads the runner-up by
          more than 2 * P_MAX the u8 labels are identical (checked on the golden's pixel grid for every
          frame and at full resolution on the last frame) — an argmax can only flip inside that margin;
          (ii) raw fraction of differing pixels per frame <= 1 % on propagated frames (measured 6e-5 at
          1 object, 6.5e-3 at 3 objects, 3e-3 at 720p / 5 objects: seeded random weights leave many
          pixels near a tie).  Frames produced by the randomly initialised FusionNet (cfg-4) sit on the
          decision boundary almost everywhere (14 % of the labels flip for max |dp| = 6.5e-3): for them
          only (i) is asserted and the raw fraction is reported.
"""
import gc
import json
import os
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mivos_b200  # noqa: E402
from mivos_b200 import _lib  # noqa: E402
from oracle import gen_golden_full as G  # noqa: E402  (checker only: clip recipes shared with the generator)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P_MAX, P_MEAN, M_FRAC, M_FRAC_FUSED = 6e-2, 2e-3, 1e-2, 1.0


def _golden(name):
    p = os.path.join(ROOT, "tests", "golden", f"full_{name}.npz")
    if not os.path.exists(p):
        pytest.skip(f"{p} not generated (python -m oracle.gen_golden_full {name})")
    from oracle import golden_io
    return golden_io.load(p)


def _net(prop_sd, dev, top_k, act):
    n = mivos_b200.PropagationNetwork(top_k=top_k, act_dtype=torch.float16 if act == "fp16" else torch.float32)
    n.load_state_dict(prop_sd, strict=True)
    return n.to(dev)


_net_cache = {}


def _cached_net(prop_sd, dev, top_k, act):
    key = (top_k, act)
    if key not in _net_cache:
        _net_cache[key] = _net(prop_sd, dev, top_k, act)
    return _net_cache[key]


def _drift(core_prob, masks, g, fused_from=None):
    """Per-frame deviations of one clip against its golden.  core_prob [(K+1),T,1,nh,nw] (device)."""
    S = int(g["stride"])
    ps = core_prob[:, :, 0, ::S, ::S].float().cpu().numpy()
    ref = g["prob_s"].astype(np.float32)
    assert ps.shape == ref.shape, (ps.shape, ref.shape)
    dp = np.abs(ps - ref)
    per_frame_dp = dp.max(axis=(0, 2, 3))
    mm = (masks != g["masks"]).reshape(masks.shape[0], -1).mean(axis=1)
    lt = int(g["last_ti"])
    ref_l = g["prob_l"].astype(np.float32)
    dl = np.abs(core_prob[:, lt, 0].float().cpu().numpy() - ref_l)
    # decided pixels: the oracle's best label leads the runner-up by more than 2 * P_MAX
    def decided_mismatch(ref, ours_lab, ref_lab):
        srt = np.sort(ref, axis=0)
        margin = srt[-1] - (srt[-2] if ref.shape[0] > 1 else 0.0)
        dec = margin > 2 * P_MAX
        return int((dec & (ours_lab != ref_lab)).sum()), int(dec.sum())
    ours_grid = np.argmax(ps, axis=0)                      # labels on the padded-frame grid [T, nh/S, nw/S]
    bad_g, n_g = decided_mismatch(ref, ours_grid, np.argmax(ref, axis=0))
    ours_last = np.argmax(core_prob[:, lt, 0].float().cpu().numpy(), axis=0)
    bad_l, n_l = decided_mismatch(ref_l, ours_last, np.argmax(ref_l, axis=0))
    return {"dp_max_per_frame": per_frame_dp.tolist(), "mask_mismatch_per_frame": mm.tolist(), "dp_mean": float(dp.mean()),
            "decided_mismatch_grid": bad_g, "decided_pixels_grid": n_g, "decided_mismatch_last": bad_l, "decided_pixels_last": n_l,
            "dp_max": float(per_frame_dp.max()), "last_frame": lt, "last_dp_max": float(dl.max()), "last_dp_mean": float(dl.mean()),
            "last_mask_mismatch": float(mm[lt]), "mask_mismatch_max": float(mm.max())}


def _report(tag, d):
    out = os.environ.get("MIVOS_DRIFT_DIR")
    if out and os.path.isdir(out):
        json.dump(d, open(os.path.join(out, f"drift_{tag}.json"), "w"))
    curve = d["dp_max_per_frame"]
    step = max(1, len(curve) // 10)
    print(f"[fullsize] {tag}: dp_max {d['dp_max']:.3e} dp_mean {d['dp_mean']:.3e} last-frame dp {d['last_dp_max']:.3e} "
          f"mask mismatch max {d['mask_mismatch_max']:.2e} last {d['last_mask_mismatch']:.2e}; decided pixels "
          f"{d['decided_pixels_grid']}+{d['decided_pixels_last']} mismatching {d['decided_mismatch_grid']}+{d['decided_mismatch_last']}; dp curve "
          + " ".join(f"{v:.1e}" for v in curve[::step]))


def _check(d, m_frac=M_FRAC):
    assert d["dp_max"] <= P_MAX and d["last_dp_max"] <= P_MAX, (d["dp_max"], d["last_dp_max"])
    assert d["dp_mean"] <= P_MEAN and d["last_dp_mean"] <= P_MEAN, (d["dp_mean"], d["last_dp_mean"])
    assert d["decided_mismatch_grid"] == 0 and d["decided_mismatch_last"] == 0, (d["decided_mismatch_grid"], d["decided_mismatch_last"])
    assert d["decided_pixels_grid"] > 0  # (the interacted frames alone are one-hot: every pixel decided)
    assert d["mask_mismatch_max"] <= m_frac, d["mask_mismatch_max"]


def _run_single(name, act, prop_sd, fuse_sd, dev, mem_profile=0):
    g = _golden(name)
    images, inter, K, top_k, mem_freq, _ = G.build_case(name)
    net = _cached_net(prop_sd, dev, top_k, act)
    fuse = None
    if len(inter) > 1:
        fuse = mivos_b200.FusionNet()
        fuse.load_state_dict(fuse_sd, strict=True)
        fuse = fuse.to(dev)
    core = mivos_b200.InferenceCore(net, fuse, images, K, mem_profile=mem_profile, mem_freq=mem_freq, device=dev)
    masks = None
    for idx, m in inter:
        masks = core.interact(m.to(dev), idx)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    assert [tuple(x) for x in g["trace"].tolist()] == core.bank_trace
    return _drift(core.prob, masks, g)


@pytest.mark.parametrize("act", ["fp16", "tf32"])
def test_cfg2_full_clip_single_session(act, prop_sd, fuse_sd, dev):
    d = _run_single("cfg2_c0", act, prop_sd, fuse_sd, dev)
    _report(f"cfg2_single_{act}", d)
    _check(d)


@pytest.mark.parametrize("act", ["fp16", "tf32"])
def test_cfg3_three_objects_topk50(act, prop_sd, fuse_sd, dev):
    d = _run_single("cfg3", act, prop_sd, fuse_sd, dev)
    _report(f"cfg3_{act}", d)
    _check(d)


@pytest.mark.parametrize("act", ["fp16", "tf32"])
def test_cfg4_fusion_two_interactions_480p(act, prop_sd, fuse_sd, dev):
    d = _run_single("cfg4", act, prop_sd, fuse_sd, dev)
    _report(f"cfg4_{act}", d)
    _check(d, m_frac=M_FRAC_FUSED)


@pytest.mark.parametrize("act", ["fp16", "tf32"])
def test_cfg5_720p_five_objects(act, prop_sd, fuse_sd, dev):
    d = _run_single("cfg5", act, prop_sd, fuse_sd, dev)
    _report(f"cfg5_{act}", d)
    _check(d)


@pytest.mark.parametrize("mem_profile", [2, 3])
def test_mem_profile_2_3_on_gpu(mem_profile, prop_sd, fuse_sd, dev):
    """q_buf_size / i_buf_size 3 and 1 (inference_core.py:44-63): query features and staged frames are
    flushed wholesale while the side stream may still read pooled buffers; results must not change."""
    d = _run_single("cfg3", "fp16", prop_sd, fuse_sd, dev, mem_profile=mem_profile)
    _report(f"cfg3_memprofile{mem_profile}_fp16", d)
    _check(d)
    d4 = _run_single("cfg4", "fp16", prop_sd, fuse_sd, dev, mem_profile=mem_profile)
    _report(f"cfg4_memprofile{mem_profile}_fp16", d4)
    _check(d4, m_frac=M_FRAC_FUSED)


@pytest.mark.parametrize("act", ["fp16", "tf32"])
def test_cfg2_timed_configuration_lanes_x_4_lockstep(act, prop_sd, fuse_sd, dev):
    """Exactly what bench.py times: its default `--clips-per-gpu` lanes (bench.CONFIGS["cfg2"]: own network object,
    CUDA stream, Python thread each), every lane advancing the four 101-frame clips (seeds 1234..1237) in lock-step, sessions
    reused across steps through InferenceCore.reset().  Every clip of every lane, on the SECOND step (after
    a reset), against the oracle's golden of that clip."""
    # the lanes x 4 101-frame sessions at once: release what the earlier cases cached (their networks' workspaces were
    # sized for the 720p / 5-object clip) so that the timed configuration has the 80 GB of an H100 to itself
    _net_cache.clear()
    gc.collect()
    torch.cuda.empty_cache()
    names = [f"cfg2_c{i}" for i in range(4)]
    gold = [_golden(n) for n in names]
    data = [G.build_case(n) for n in names]
    results = {}

    class Lane:
        def __init__(self, i):
            self.i = i
            self.net = _net(prop_sd, dev, 20, act)
            self.stream = torch.cuda.Stream(device=dev)
            self.cores = [mivos_b200.InferenceCore(self.net, None, d[0], 1, mem_profile=0, mem_freq=5, device=dev) for d in data]
            self.err = None

        def run(self):
            try:
                torch.cuda.set_device(dev)
                torch.set_grad_enabled(False)
                with torch.cuda.stream(self.stream):
                    for step in range(2):
                        for c in self.cores:
                            c.reset()
                        masks = mivos_b200.LockstepSession(self.cores).interact([d[1][0][1].to(dev) for d in data], 0)
                    self.stream.synchronize()
                results[self.i] = masks
            except Exception as e:  # surfaced in the main thread
                self.err = e

    import bench
    n_lanes, n_clips = bench.CONFIGS["cfg2"]["lanes"], bench.CONFIGS["cfg2"]["lockstep"]
    assert n_clips == len(names)  # the four clip seeds of a lane are the goldens above
    lanes = [Lane(i) for i in range(n_lanes)]
    for ln in lanes:  # graph capture is single-threaded (as in bench.py's warm-up), then all lanes concurrently
        ln.run()
        assert ln.err is None, ln.err
    threads = [threading.Thread(target=ln.run) for ln in lanes]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    worst = None
    for ln in lanes:
        assert ln.err is None, ln.err
        for c, (core, g) in enumerate(zip(ln.cores, gold)):
            assert [tuple(x) for x in g["trace"].tolist()] == core.bank_trace
            d = _drift(core.prob, results[ln.i][c], g)
            _report(f"cfg2_lane{ln.i}_clip{c}_{act}", d)
            _check(d)
            if worst is None or d["dp_max"] > worst["dp_max"]:
                worst = d
    print(f"[fullsize] {n_lanes}x4 lock-step {act}: worst clip dp_max {worst['dp_max']:.3e}, mask mismatch {worst['mask_mismatch_max']:.2e}")
