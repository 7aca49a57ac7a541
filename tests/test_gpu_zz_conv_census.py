"""GPU: the conv census (tests/conv_census.py) and the memory census (tests/memory_census.py) over real sessions —
every mivos_conv_gemm launch, memory read and bank write the engines make, at the shapes, plans and layouts production
picks, checked on its own operands against float64 restatements of the ABI contracts with the bounds of DESIGN.md
section 6.  Each launch signature is checked once; `-s` prints the tables of checked launches.

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
  objects40_112  InferenceCore, K = 40 (object chunks 14 + 13 + 13), 112x176, two interactions, the second fused
  objects17_480  InferenceCore, K = 17 (chunks 9 + 8), 480x864, one interaction, fp16
  ragged112  LockstepSession(ragged=True), 4 clips x K = 2 of the lengths, mem_freq and interaction frames of
             MIXED in tests/test_gpu_mixed_objects.py, a second interaction fusing on some clips: prefix ticks
  ragged480  the same at 480x864 with 3 clips and one interaction, fp16
  mixed112   LockstepSession(mixed_objects=True) over the MIXED clips (K = 1, 3, 2, 5), two interactions
  dense_wide160  top_k=None and top_k=100 networks at 160x224: one InferenceCore, one ragged and one mixed session
             each, so that all nine read forms run
The session scenarios first run as users run them (graphs, overlapped lanes, no host synchronisation), then eagerly
under the census: probabilities and masks must be equal, so the checked launches produced exactly what users get."""
import contextlib
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mivos_b200  # noqa: E402
from mivos_b200 import _lib  # noqa: E402
from oracle import weights as Wt  # noqa: E402

import conv_census as CC  # noqa: E402
import memory_census as MC  # noqa: E402
from mivos_b200.engine import object_chunks  # noqa: E402
from test_gpu_mixed_objects import MIXED  # noqa: E402

ACTS = {"fp16": torch.float16, "tf32": torch.float32}
H100_SXM_SMS = 132


@pytest.fixture(scope="module")
def census():
    c = CC.Census()
    yield c
    print("\n" + c.table() + "\n" + c.summary())


@pytest.fixture(scope="module")
def memory():
    m = MC.MemoryCensus()
    yield m
    print("\n" + m.table() + "\n" + m.summary())


@contextlib.contextmanager
def _recording(rec, scenario, net=None, fuse=None):
    """Both censuses over the block when rec = (conv census, memory census); production (no census) when None."""
    if rec is None:
        yield
        return
    census, memory = rec
    if net is not None:
        _label(census, net, fuse)
    with census.record(scenario), memory.record(scenario):
        yield


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


def _session(prop_sd, fuse_sd, dev, act, clip, interactions, K, fuse=True, census=None, scenario=None, top_k=20,
             **core_kw):
    """One InferenceCore session on fresh networks; under the censuses when given them (eager launches)."""
    net, f = _nets(prop_sd, fuse_sd, dev, act, top_k=top_k, fuse=fuse)
    core = mivos_b200.InferenceCore(net, f, clip, K, device=dev, **core_kw)
    masks = []
    with _recording(census, scenario, net, f):
        for idx, m in interactions:
            masks.append(core.interact(m.to(dev), idx).copy())
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    return core.prob.clone(), masks


def _production_then_census(monkeypatch, census, memory, scenario, run):
    """run(rec) -> (probabilities, masks): as users run it, then eagerly under both censuses; the same bits."""
    t0 = time.time()
    monkeypatch.setenv("MIVOS_GRAPH", "1")
    want = run(None)
    monkeypatch.setenv("MIVOS_GRAPH", "0")
    got = run((census, memory))
    for a, b in zip(want[0], got[0]):
        assert torch.equal(a, b), f"{scenario}: probabilities of the census run differ from production"
    for a, b in zip(want[1], got[1]):
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), f"{scenario}: masks differ from production"
    print(f"\n[census] {scenario}: {census.seen[scenario]} conv launches seen, {census.checked[scenario]} checked; "
          f"{memory.seen[scenario]} memory launches seen, {memory.checked[scenario]} checked; {time.time() - t0:.1f} s")
    assert census.checked[scenario] > 0 and memory.checked[scenario] > 0


def _second_mask(K, H, W, seed):
    _, m = Wt.synthetic_clip(1, H, W, K, seed=seed)
    return m.flip(-1).contiguous()


@pytest.mark.parametrize("act", list(ACTS))
def test_census_core480_two_interactions(act, prop_sd, fuse_sd, dev, census, memory, monkeypatch):
    H, W, T, K = 480, 864, 10, 2
    clip, m0 = Wt.synthetic_clip(T, H, W, K, seed=480)
    inter = [(0, m0), (5, _second_mask(K, H, W, 481))]
    sc = f"core480_{act}"

    def run(c):
        p, m = _session(prop_sd, fuse_sd, dev, act, clip, inter, K, census=c, scenario=sc, mem_freq=5)
        return [p], [m]
    _production_then_census(monkeypatch, census, memory, sc, run)


@pytest.mark.parametrize("act", list(ACTS))
def test_census_lockstep480_four_clips(act, prop_sd, fuse_sd, dev, census, memory, monkeypatch):
    H, W, T, C, K = 480, 864, 4, 4, 1
    clips = [Wt.synthetic_clip(T, H, W, K, seed=500 + i) for i in range(C)]
    sc = f"lock480_{act}"

    def run(c):
        net, _ = _nets(prop_sd, fuse_sd, dev, act, fuse=False)
        cores = [mivos_b200.InferenceCore(net, None, im, K, mem_freq=2, device=dev) for im, _ in clips]
        sess = mivos_b200.LockstepSession(cores)
        with _recording(c, sc, net):
            out = sess.interact([m for _, m in clips], 0)
        torch.cuda.synchronize()
        _lib.poll_kernel_error()
        return [x.prob.clone() for x in cores], [[o.copy() for o in out]]
    _production_then_census(monkeypatch, census, memory, sc, run)


@pytest.mark.parametrize("act", list(ACTS))
def test_census_core112_three_objects(act, prop_sd, fuse_sd, dev, census, memory, monkeypatch):
    H, W, T, K = 112, 176, 4, 3
    clip, m0 = Wt.synthetic_clip(T, H, W, K, seed=112)
    sc = f"core112_{act}"

    def run(c):
        p, m = _session(prop_sd, fuse_sd, dev, act, clip, [(0, m0)], K, fuse=False, census=c, scenario=sc, mem_freq=2)
        return [p], [m]
    _production_then_census(monkeypatch, census, memory, sc, run)


@pytest.mark.parametrize("act", list(ACTS))
def test_census_core1080_fused(act, prop_sd, fuse_sd, dev, census, memory, monkeypatch):
    H, W, T, K = 1080, 1920, 3, 2
    clip, m0 = Wt.synthetic_clip(T, H, W, K, seed=1080)
    inter = [(0, m0), (2, _second_mask(K, H, W, 1081))]
    sc = f"core1080_{act}"

    def run(c):
        p, m = _session(prop_sd, fuse_sd, dev, act, clip, inter, K, census=c, scenario=sc, mem_freq=5)
        return [p], [m]
    _production_then_census(monkeypatch, census, memory, sc, run)


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("n,H,W", [(2, 480, 864), (1, 1088, 1920)], ids=["480p_n2", "1080p_n1"])
def test_census_s2m(act, n, H, W, dev, census, memory):
    net = mivos_b200.S2MNetwork(act_dtype=ACTS[act])
    net.load_state_dict(Wt.make_s2m_state_dict(), strict=True)
    net = net.to(dev)
    census.label(net.engine().pc, "s2m.")
    g = torch.Generator().manual_seed(H + n)
    x = torch.cat([torch.randn((n, 3, H, W), generator=g), (torch.rand((n, 3, H, W), generator=g) > 0.7).float()], 1)
    sc = f"s2m{H}_n{n}_{act}"
    t0 = time.time()
    with _recording((census, memory), sc):
        p = net.forward_sigmoid(x.to(dev))
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    assert bool(torch.isfinite(p).all())
    print(f"\n[census] {sc}: {census.seen[sc]} launches seen, {census.checked[sc]} checked, {time.time() - t0:.1f} s")
    assert census.checked[sc] > 0


def test_census_core4k_fp16(prop_sd, fuse_sd, dev, census, memory, monkeypatch):
    """Query pass, memorize and one segment at 4K (frame 1 propagated from the interaction at frame 0)."""
    monkeypatch.setenv("MIVOS_GRAPH", "0")
    H, W, T, K = 2160, 3840, 2, 1
    clip, m0 = Wt.synthetic_clip(T, H, W, K, seed=2160)
    t0 = time.time()
    prob, _ = _session(prop_sd, fuse_sd, dev, "fp16", clip, [(0, m0)], K, fuse=False, census=(census, memory),
                       scenario="core4k_fp16", mem_profile=2)
    p = prob[:, 1, 0]
    assert bool(torch.isfinite(p).all()) and float((p.sum(0) - 1).abs().max()) <= 1e-5
    print(f"\n[census] core4k_fp16: {census.seen['core4k_fp16']} conv launches seen, {census.checked['core4k_fp16']} "
          f"checked; {memory.seen['core4k_fp16']} memory launches seen, {memory.checked['core4k_fp16']} checked; "
          f"{time.time() - t0:.1f} s")


# ---- object chunks, ragged and mixed-object lock-step, dense and wide reads -----------------------------------------

@pytest.mark.parametrize("act", list(ACTS))
def test_census_objects40_112(act, prop_sd, fuse_sd, dev, census, memory, monkeypatch):
    """40 objects: memorize and decoder in chunks of 14 + 13 + 13 maps, each chunk reading its bank slice and writing
    its slice of the 40-object logits map; the second interaction fuses."""
    H, W, T, K = 112, 176, 4, 40
    clip, m0 = Wt.synthetic_clip(T, H, W, K, seed=4040)
    inter = [(0, m0), (3, _second_mask(K, H, W, 4041))]
    sc = f"objects40_112_{act}"

    def run(c):
        p, m = _session(prop_sd, fuse_sd, dev, act, clip, inter, K, census=c, scenario=sc, mem_freq=2)
        return [p], [m]
    _production_then_census(monkeypatch, census, memory, sc, run)


def test_census_objects17_480_fp16(prop_sd, fuse_sd, dev, census, memory, monkeypatch):
    H, W, T, K = 480, 864, 3, 17
    clip, m0 = Wt.synthetic_clip(T, H, W, K, seed=1717)
    sc = "objects17_480_fp16"

    def run(c):
        p, m = _session(prop_sd, fuse_sd, dev, "fp16", clip, [(0, m0)], K, fuse=False, census=c, scenario=sc,
                        mem_freq=2)
        return [p], [m]
    _production_then_census(monkeypatch, census, memory, sc, run)


def _lockstep(prop_sd, fuse_sd, dev, act, rec, sc, H, W, plans, rounds, *, top_k=20, fuse=True, **sess_kw):
    """A LockstepSession over clips of plans (objects, length, mem_freq, first interaction, second interaction):
    `rounds` interactions, the second with mirrored masks.  Returns (probabilities, masks of each round)."""
    net, f = _nets(prop_sd, fuse_sd, dev, act, top_k=top_k, fuse=fuse)
    clips = [Wt.synthetic_clip(t, H, W, k, seed=40 + i) for i, (k, t, *_r) in enumerate(plans)]
    cores = [mivos_b200.InferenceCore(net, f, img, p[0], mem_freq=p[2], device=dev) for (img, _m), p in zip(clips, plans)]
    sess = mivos_b200.LockstepSession(cores, **sess_kw)
    outs = []
    with _recording(rec, sc, net, f):
        for r in range(rounds):
            masks = [(m if r == 0 else m.flip(-1)).contiguous() for _img, m in clips]
            outs.append([o.copy() for o in sess.interact(masks, [p[3 + r] for p in plans])])
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    return [c.prob.clone() for c in cores], outs


def _ragged_plans(K, clips):
    return [(K,) + tuple(p[1:]) for p in MIXED[:clips]]


@pytest.mark.parametrize("act", list(ACTS))
def test_census_ragged112(act, prop_sd, fuse_sd, dev, census, memory, monkeypatch):
    sc = f"ragged112_{act}"
    _production_then_census(monkeypatch, census, memory, sc, lambda c: _lockstep(
        prop_sd, fuse_sd, dev, act, c, sc, 112, 176, _ragged_plans(2, 4), 2, ragged=True))


def test_census_ragged480_fp16(prop_sd, fuse_sd, dev, census, memory, monkeypatch):
    sc = "ragged480_fp16"
    _production_then_census(monkeypatch, census, memory, sc, lambda c: _lockstep(
        prop_sd, fuse_sd, dev, "fp16", c, sc, 480, 864, _ragged_plans(2, 3), 1, fuse=False, ragged=True))


@pytest.mark.parametrize("act", list(ACTS))
def test_census_mixed112(act, prop_sd, fuse_sd, dev, census, memory, monkeypatch):
    sc = f"mixed112_{act}"
    _production_then_census(monkeypatch, census, memory, sc, lambda c: _lockstep(
        prop_sd, fuse_sd, dev, act, c, sc, 112, 176, MIXED, 2, mixed_objects=True))


@pytest.mark.parametrize("act", list(ACTS))
def test_census_dense_wide160(act, prop_sd, fuse_sd, dev, census, memory, monkeypatch):
    """top_k=None and top_k=100 at 160x224 (hw = 140 >= 100 from the first frame): one InferenceCore, one ragged and
    one mixed session each — the scalar, per-set and grouped dense and wide reads."""
    H, W = 160, 224
    sc = f"dense_wide160_{act}"
    clip, m0 = Wt.synthetic_clip(5, H, W, 2, seed=160)

    def run(c):
        probs, masks = [], []
        for top_k in (None, 100):
            p, m = _session(prop_sd, fuse_sd, dev, act, clip, [(1, m0)], 2, fuse=False, census=c, scenario=sc,
                            top_k=top_k, mem_freq=2)
            probs.append(p)
            masks.append(m)
            for kw in (dict(ragged=True), dict(mixed_objects=True)):
                plans = _ragged_plans(2, 4) if "ragged" in kw else MIXED
                p, m = _lockstep(prop_sd, fuse_sd, dev, act, c, sc, H, W, plans, 1, top_k=top_k, fuse=False, **kw)
                probs += p
                masks += m
        return probs, masks
    _production_then_census(monkeypatch, census, memory, sc, run)


SCENARIOS = ["core480_fp16", "core480_tf32", "lock480_fp16", "lock480_tf32", "core112_fp16", "core112_tf32",
             "core1080_fp16", "core1080_tf32", "s2m480_n2_fp16", "s2m480_n2_tf32", "s2m1088_n1_fp16",
             "s2m1088_n1_tf32", "core4k_fp16", "objects40_112_fp16", "objects40_112_tf32", "objects17_480_fp16",
             "ragged112_fp16", "ragged112_tf32", "ragged480_fp16", "mixed112_fp16", "mixed112_tf32",
             "dense_wide160_fp16", "dense_wide160_tf32"]
CHUNK_NS = {n for K in (40, 17) for _k0, n in object_chunks(K)}
LOCKSTEP = ("lock480", "ragged", "mixed", "dense_wide")


def coverage(records):
    """Facts the conv census must contain (taken from mivos_conv_plan at 132 SMs): fact -> present."""
    def has(f):
        return any(f(r) for r in records)
    facts = {f"taps {t}": has(lambda r, t=t: r["taps"] == t) for t in (1, 4, 9)}
    facts.update({f"BN {b}": has(lambda r, b=b: r["bn"] == b) for b in (32, 64, 128, 256)})
    for name, f16 in (("fp16", True), ("tf32", False)):
        facts[f"S >= 2, {name}"] = has(lambda r, f16=f16: r["s"] >= 2 and r["f16"] == f16)
        facts[f"S >= 2 with a residual, {name}"] = has(lambda r, f16=f16: r["s"] >= 2 and r["f16"] == f16 and r["res"])
        facts[f"S >= 2 into out_coff > 0, {name}"] = has(lambda r, f16=f16: r["s"] >= 2 and r["f16"] == f16 and r["out_coff"] > 0)
        facts[f"2 CTAs per SM, {name}"] = has(lambda r, f16=f16: r["ctas"] == 2 and r["f16"] == f16)
    facts["2 CTAs per SM with a residual"] = has(lambda r: r["ctas"] == 2 and r["res"])
    facts["pre-gathered operand under split-K"] = has(lambda r: r["mat"] and r["taps"] == 1 and r["s"] >= 2)
    facts["fp32 output from fp16 operands"] = has(lambda r: r["f16"] and not r["out_f16"])
    facts["dual output"] = has(lambda r: r["dual"])
    facts["n >= 8"] = has(lambda r: r["n"] >= 8)
    facts["a chunk batch (K > 16)"] = has(lambda r: r["scenario"].startswith("objects") and r["n"] in CHUNK_NS)
    facts["a prefix tick"] = has(lambda r: r["scenario"].startswith(LOCKSTEP) and r["n"] < r["alloc_maps"])
    return facts


def memory_coverage(reads, writes):
    """Facts the memory census must contain: fact -> present."""
    def has(f, rs=reads):
        return any(f(r) for r in rs)
    facts = {f"{form} checked": has(lambda r, form=form: r["form"] == form) for form in MC.READS}
    facts["fp16 cat"] = has(lambda r: r["f16"])
    facts["fp32 cat"] = has(lambda r: not r["f16"])
    facts["q_div > 0"] = has(lambda r: r["layout"] == "scalar" and r["q_div"] > 0)
    facts["a device count below capacity"] = has(lambda r: r["device_count"] and min(r["live"]) < r["cap"])
    facts["counts that differ within a sets / groups launch"] = has(
        lambda r: r["layout"] != "scalar" and len(set(r["counts"])) > 1)
    facts["a one-object group"] = has(
        lambda r: r["layout"] == "groups" and any(b - a == 1 for a, b in zip(r["first"], r["first"][1:])))
    facts["a bank slice not starting at object 0"] = has(lambda r: r["bank0"] > 0)
    facts["a live count not a multiple of 32"] = has(lambda r: any(n % 32 for n in r["live"] if n))
    for form in MC.WRITES:
        facts[f"{form} checked"] = has(lambda r, form=form: r["form"] == form, writes)
    return facts


def test_census_coverage(census, memory, dev):
    ran = set(census.seen)
    missing_runs = [s for s in SCENARIOS if s not in ran]
    if missing_runs:
        pytest.skip(f"scenarios not run in this session: {missing_runs}")
    facts = coverage(census.records)
    facts.update({f"memory: {k}": v for k, v in memory_coverage(memory.records, memory.writes).items()})
    missing = [k for k, v in facts.items() if not v]
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    st = [r["stats"] for r in memory.records if r["stats"]]
    print(f"\n[census] {len(census.records)} conv launches checked of {sum(census.seen.values())}; worst err/bound "
          f"{max(r['ratio'] for r in census.records):.3g}; {len(memory.records)} reads and {len(memory.writes)} bank "
          f"writes checked of {sum(memory.seen.values())} memory launches; worst read err/bound "
          f"{max(r['ratio'] for r in memory.records):.3g}; TF32 path: {sum(x[2] for x in st)} of "
          f"{sum(r['maps'] * r['hw'] for r in memory.records if r['stats'])} queries on the exact fallback; {sms} SMs; "
          f"{len(facts)} facts, missing: {missing or 'none'}")
    if sms == H100_SXM_SMS:
        assert not missing, f"the census lost coverage: {missing}"
