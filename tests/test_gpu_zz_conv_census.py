"""GPU: the conv census (tests/conv_census.py) over real sessions — every mivos_conv_gemm launch the engines make, at
the shapes and plans production picks, checked on its own operands against the float64 ABI contract with the bound of
DESIGN.md section 6.  Each launch signature is checked once; `-s` prints the table of checked launches.

Scenarios (seeded weights and clips of oracle.weights), on fp16 and TF32 unless stated:
  core480    InferenceCore, 480x864, K = 2, top-k 20, 10 frames (a full query chunk of 8), interactions at frames 0
             and 5 (the second pass fuses): query chunk N = 8, memorize n = 2, segment, decoder split-K with a
             residual, FusionNet (TF32)
  lock480    LockstepSession of 4 clips x K = 1 at 480x864: encode_memory / segment at C = 4, n = 4
  core112    InferenceCore, 112x176, K = 3: 7x11 maps at 1/16, one partial M tile spanning images
  core1080   InferenceCore, 1088x1920 (a 1080p clip), K = 2, 3 frames, a fused second interaction: S = 3 plans
  s2m        the S2M network at 480x864, n = 2, and at 1088x1920, n = 1: im2col stem, dilated K = 18432 under
             S = 8 into the windows of the concat map, the 304 -> 320 head
  core4k     2160x3840, K = 1, fp16: query pass, memorize and one segment (row-sampled)
The session scenarios first run as users run them (graphs, overlapped lanes, no host synchronisation), then eagerly
under the census: probabilities and masks must be equal, so the checked launches produced exactly what users get."""
import os
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mivos_b200  # noqa: E402
from mivos_b200 import _lib  # noqa: E402
from oracle import weights as Wt  # noqa: E402

import conv_census as CC  # noqa: E402

ACTS = {"fp16": torch.float16, "tf32": torch.float32}
H100_SXM_SMS = 132


@pytest.fixture(scope="module")
def census():
    c = CC.Census()
    yield c
    print("\n" + c.table() + "\n" + c.summary())


def _nets(prop_sd, fuse_sd, dev, act, top_k=20, fuse=True):
    net = mivos_b200.PropagationNetwork(top_k=top_k, act_dtype=ACTS[act])
    net.load_state_dict(prop_sd, strict=True)
    net = net.to(dev)
    f = None
    if fuse:
        f = mivos_b200.FusionNet()
        f.load_state_dict(fuse_sd, strict=True)
        f = f.to(dev)
    return net, f


def _label(census, net, fuse):
    census.label(net.engine().pc)
    if fuse is not None:
        census.label(fuse.engine().pc, "fusion.")


def _session(prop_sd, fuse_sd, dev, act, clip, interactions, K, fuse=True, census=None, scenario=None, **core_kw):
    """One InferenceCore session on fresh networks; under the census when given one (eager launches)."""
    net, f = _nets(prop_sd, fuse_sd, dev, act, fuse=fuse)
    core = mivos_b200.InferenceCore(net, f, clip, K, device=dev, **core_kw)
    masks = []
    if census is None:
        for idx, m in interactions:
            masks.append(core.interact(m.to(dev), idx).copy())
    else:
        _label(census, net, f)
        with census.record(scenario):
            for idx, m in interactions:
                masks.append(core.interact(m.to(dev), idx).copy())
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    return core.prob.clone(), masks


def _production_then_census(monkeypatch, census, scenario, run):
    """run(census) -> (probabilities, masks): as users run it, then eagerly under the census; the same bits."""
    t0 = time.time()
    monkeypatch.setenv("MIVOS_GRAPH", "1")
    want = run(None)
    monkeypatch.setenv("MIVOS_GRAPH", "0")
    got = run(census)
    for a, b in zip(want[0], got[0]):
        assert torch.equal(a, b), f"{scenario}: probabilities of the census run differ from production"
    for a, b in zip(want[1], got[1]):
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), f"{scenario}: masks differ from production"
    print(f"\n[census] {scenario}: {census.seen[scenario]} launches seen, {census.checked[scenario]} checked, "
          f"{time.time() - t0:.1f} s")
    assert census.checked[scenario] > 0


def _second_mask(K, H, W, seed):
    _, m = Wt.synthetic_clip(1, H, W, K, seed=seed)
    return m.flip(-1).contiguous()


@pytest.mark.parametrize("act", list(ACTS))
def test_census_core480_two_interactions(act, prop_sd, fuse_sd, dev, census, monkeypatch):
    H, W, T, K = 480, 864, 10, 2
    clip, m0 = Wt.synthetic_clip(T, H, W, K, seed=480)
    inter = [(0, m0), (5, _second_mask(K, H, W, 481))]
    sc = f"core480_{act}"

    def run(c):
        p, m = _session(prop_sd, fuse_sd, dev, act, clip, inter, K, census=c, scenario=sc, mem_freq=5)
        return [p], [m]
    _production_then_census(monkeypatch, census, sc, run)


@pytest.mark.parametrize("act", list(ACTS))
def test_census_lockstep480_four_clips(act, prop_sd, fuse_sd, dev, census, monkeypatch):
    H, W, T, C, K = 480, 864, 4, 4, 1
    clips = [Wt.synthetic_clip(T, H, W, K, seed=500 + i) for i in range(C)]
    sc = f"lock480_{act}"

    def run(c):
        net, _ = _nets(prop_sd, fuse_sd, dev, act, fuse=False)
        cores = [mivos_b200.InferenceCore(net, None, im, K, mem_freq=2, device=dev) for im, _ in clips]
        sess = mivos_b200.LockstepSession(cores)
        if c is None:
            out = sess.interact([m for _, m in clips], 0)
        else:
            _label(c, net, None)
            with c.record(sc):
                out = sess.interact([m for _, m in clips], 0)
        torch.cuda.synchronize()
        _lib.poll_kernel_error()
        return [x.prob.clone() for x in cores], [[o.copy() for o in out]]
    _production_then_census(monkeypatch, census, sc, run)


@pytest.mark.parametrize("act", list(ACTS))
def test_census_core112_three_objects(act, prop_sd, fuse_sd, dev, census, monkeypatch):
    H, W, T, K = 112, 176, 4, 3
    clip, m0 = Wt.synthetic_clip(T, H, W, K, seed=112)
    sc = f"core112_{act}"

    def run(c):
        p, m = _session(prop_sd, fuse_sd, dev, act, clip, [(0, m0)], K, fuse=False, census=c, scenario=sc, mem_freq=2)
        return [p], [m]
    _production_then_census(monkeypatch, census, sc, run)


@pytest.mark.parametrize("act", list(ACTS))
def test_census_core1080_fused(act, prop_sd, fuse_sd, dev, census, monkeypatch):
    H, W, T, K = 1080, 1920, 3, 2
    clip, m0 = Wt.synthetic_clip(T, H, W, K, seed=1080)
    inter = [(0, m0), (2, _second_mask(K, H, W, 1081))]
    sc = f"core1080_{act}"

    def run(c):
        p, m = _session(prop_sd, fuse_sd, dev, act, clip, inter, K, census=c, scenario=sc, mem_freq=5)
        return [p], [m]
    _production_then_census(monkeypatch, census, sc, run)


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("n,H,W", [(2, 480, 864), (1, 1088, 1920)], ids=["480p_n2", "1080p_n1"])
def test_census_s2m(act, n, H, W, dev, census):
    net = mivos_b200.S2MNetwork(act_dtype=ACTS[act])
    net.load_state_dict(Wt.make_s2m_state_dict(), strict=True)
    net = net.to(dev)
    census.label(net.engine().pc, "s2m.")
    g = torch.Generator().manual_seed(H + n)
    x = torch.cat([torch.randn((n, 3, H, W), generator=g), (torch.rand((n, 3, H, W), generator=g) > 0.7).float()], 1)
    sc = f"s2m{H}_n{n}_{act}"
    t0 = time.time()
    with census.record(sc):
        p = net.forward_sigmoid(x.to(dev))
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    assert bool(torch.isfinite(p).all())
    print(f"\n[census] {sc}: {census.seen[sc]} launches seen, {census.checked[sc]} checked, {time.time() - t0:.1f} s")
    assert census.checked[sc] > 0


def test_census_core4k_fp16(prop_sd, fuse_sd, dev, census, monkeypatch):
    """Query pass, memorize and one segment at 4K (frame 1 propagated from the interaction at frame 0)."""
    monkeypatch.setenv("MIVOS_GRAPH", "0")
    H, W, T, K = 2160, 3840, 2, 1
    clip, m0 = Wt.synthetic_clip(T, H, W, K, seed=2160)
    t0 = time.time()
    prob, _ = _session(prop_sd, fuse_sd, dev, "fp16", clip, [(0, m0)], K, fuse=False, census=census,
                       scenario="core4k_fp16", mem_profile=2)
    p = prob[:, 1, 0]
    assert bool(torch.isfinite(p).all()) and float((p.sum(0) - 1).abs().max()) <= 1e-5
    print(f"\n[census] core4k_fp16: {census.seen['core4k_fp16']} launches seen, {census.checked['core4k_fp16']} checked, "
          f"{time.time() - t0:.1f} s")


SCENARIOS = ["core480_fp16", "core480_tf32", "lock480_fp16", "lock480_tf32", "core112_fp16", "core112_tf32",
             "core1080_fp16", "core1080_tf32", "s2m480_n2_fp16", "s2m480_n2_tf32", "s2m1088_n1_fp16",
             "s2m1088_n1_tf32", "core4k_fp16"]


def coverage(records):
    """Facts the census must contain (taken from mivos_conv_plan at 132 SMs): fact -> present."""
    def has(f):
        return any(f(r) for r in records)
    facts = {f"taps {t}": has(lambda r, t=t: r["taps"] == t) for t in (1, 4, 9)}
    facts.update({f"BN {b}": has(lambda r, b=b: r["bn"] == b) for b in (32, 64, 128, 256)})
    for name, f16 in (("fp16", True), ("tf32", False)):
        facts[f"S >= 2, {name}"] = has(lambda r, f16=f16: r["s"] >= 2 and r["f16"] == f16)
        facts[f"S >= 2 with a residual, {name}"] = has(lambda r, f16=f16: r["s"] >= 2 and r["f16"] == f16 and r["res"])
        facts[f"S >= 2 into out_coff > 0, {name}"] = has(lambda r, f16=f16: r["s"] >= 2 and r["f16"] == f16 and r["out_coff"] > 0)
    facts["pre-gathered operand under split-K"] = has(lambda r: r["mat"] and r["taps"] == 1 and r["s"] >= 2)
    facts["fp32 output from fp16 operands"] = has(lambda r: r["f16"] and not r["out_f16"])
    facts["dual output"] = has(lambda r: r["dual"])
    facts["n >= 8"] = has(lambda r: r["n"] >= 8)
    return facts


def test_census_coverage(census, dev):
    ran = set(census.seen)
    missing_runs = [s for s in SCENARIOS if s not in ran]
    if missing_runs:
        pytest.skip(f"scenarios not run in this session: {missing_runs}")
    facts = coverage(census.records)
    missing = [k for k, v in facts.items() if not v]
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    print(f"\n[census] {len(census.records)} launches checked of {sum(census.seen.values())}; worst err/bound "
          f"{max(r['ratio'] for r in census.records):.3g}; {sms} SMs; missing facts: {missing or 'none'}")
    if sms == H100_SXM_SMS:
        assert not missing, f"the census lost coverage: {missing}"
