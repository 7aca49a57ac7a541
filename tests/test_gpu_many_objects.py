"""GPU: clips of 17 to 255 objects.  The plane kernels of the aggregation (mivos_*_planes) against float64 at the
bound of tests/test_gpu_ops_ragged.py (whose background term grows as K u) and bit for bit against the register
kernels at K <= 16; the object-range stem gather against float64 and bit for bit against the whole-clip gather; the
object-chunked InferenceCore against the goldens of the UNMODIFIED reference (oracle/gen_golden_objects.py) on the
TF32 and the fp16 path at the tolerances of tests/test_gpu_network.py; graph replay against eager launches."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mivos_b200  # noqa: E402
from mivos_b200 import _lib, ops  # noqa: E402
from mivos_b200.engine import object_chunks  # noqa: E402
from oracle import gen_golden_objects as GO  # noqa: E402  (input recipes of the goldens)
from oracle import weights as Wt  # noqa: E402  (synthetic clips only)
from op_references import (U, _bilinear, _sum_and_range, aggregate_reference, stem_reference,  # noqa: E402,F401
                           stem_tolerance)
from test_gpu_ops_ragged import NAN, SENT, _check, _halo, _logits  # noqa: E402

P_MAX, P_MEAN = 3e-2, 1e-3
SHAPES = ((1, 1), (3, 5), (7, 9))  # (h4, w4): ragged pixel counts, 16 to 1008 pixels per plane


def _fused(K, groups, h4, w4, planes, dev, seed):
    lg = _logits(groups, K, h4, w4, seed).to(dev)
    halo = _halo(lg[:, None], 7, 5, fill=NAN)  # channel 5 of a 7-channel map, NaN everywhere else
    H, W = 4 * h4, 4 * w4
    raw = torch.full((groups * K, 1, H, W), SENT, device=dev)
    prob = torch.full(((groups,) if groups > 1 else ()) + (K + 1, 1, H, W), SENT, device=dev)
    fn = ops.upsample4x_sigmoid_aggregate_planes if planes else ops.upsample4x_sigmoid_aggregate
    fn(halo, K, h4, w4, coff=5, raw_out=raw, prob_out=prob, groups=groups)
    return lg, raw, prob


def _probs(K, n, dev, seed):
    """[K,1,n] probabilities with exact 0 / 1 (the clamp limits) and values next to them."""
    g = torch.Generator().manual_seed(seed)
    p = torch.rand((K, 1, n), generator=g)
    pick = torch.randint(0, 6, p.shape, generator=g)
    p = torch.where(pick == 0, torch.zeros_like(p), torch.where(pick == 1, torch.ones_like(p), p))
    p = torch.where(pick == 2, torch.full_like(p, 1e-8), torch.where(pick == 3, torch.full_like(p, 1 - 2 ** -24), p))
    return p.to(dev).contiguous()


# ------------------------------------------------------------------------------------------------ aggregation
@pytest.mark.parametrize("K", [1, 3, 16])
def test_plane_kernels_equal_register_kernels(dev, K):
    """At K <= 16 the plane kernels give the register kernels' bits: the operation order was kept."""
    for groups in (1, 3):
        for h4, w4 in SHAPES:
            _, raw0, prob0 = _fused(K, groups, h4, w4, False, dev, K * 10 + groups + h4)
            _, raw1, prob1 = _fused(K, groups, h4, w4, True, dev, K * 10 + groups + h4)
            assert torch.equal(raw0, raw1) and torch.equal(prob0, prob1), (K, groups, h4, w4)
    p = _probs(K, 997, dev, K)
    for keep_bg in (True, False):
        for hard in (False, True):
            for const_bg in (False, True):
                a = ops.aggregate_wbg(p, keep_bg=keep_bg, hard=hard, const_bg=const_bg)
                b = ops.aggregate_wbg_planes(p, keep_bg=keep_bg, hard=hard, const_bg=const_bg)
                assert torch.equal(a, b), (K, keep_bg, hard, const_bg)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()


@pytest.mark.parametrize("K", [17, 31, 64, 255])
def test_plane_kernels_against_float64(dev, K):
    for groups in (1, 2):
        for h4, w4 in SHAPES:
            lg, raw, prob = _fused(K, groups, h4, w4, True, dev, K * 10 + groups + h4)
            torch.cuda.synchronize()
            H, W = 4 * h4, 4 * w4
            tag = f"K={K} G={groups} {h4}x{w4}"
            v = _bilinear(lg[:, None], H, W)
            p = torch.sigmoid(v)
            rb = p * (1 - p) * 4 * U * _bilinear(lg.abs()[:, None], H, W) + p * (2 * U + 4 * U * (1 - p))
            _check(f"upsample4x_planes raw {tag}", raw, p, rb)
            pr, pg = raw.reshape(groups, K, H, W), prob.reshape(groups, K + 1, H, W)
            for gi in range(groups):
                o, ob, _ = aggregate_reference(pr[gi])
                _check(f"upsample4x_planes prob {tag} group {gi}", pg[gi], o, ob)
                _sum_and_range(f"upsample4x_planes prob {tag} group {gi}", pg[gi], K)
    for n in (1, 37, 1009):
        pk = _probs(K, n, dev, K + n)
        for keep_bg in (True, False):
            for const_bg in (False, True):
                got = ops.aggregate_wbg_planes(pk, keep_bg=keep_bg, const_bg=const_bg)
                o, ob, lgt = aggregate_reference(pk[:, 0], const_bg)
                what = f"aggregate_wbg_planes K={K} n={n} keep_bg={keep_bg} const_bg={const_bg}"
                _check(what, got[:, 0], o if keep_bg else o[1:], ob if keep_bg else ob[1:])
                if keep_bg:
                    _sum_and_range(what, got[:, 0], K)
                hard = ops.aggregate_wbg_planes(pk, keep_bg=True, hard=True, const_bg=const_bg)[:, 0]
                hl = 1000 * lgt
                top2 = hl.topk(2, 0).values
                clear = top2[0] - top2[1] > 20
                onehot = torch.nn.functional.one_hot(hl.argmax(0), K + 1).t().double()
                tol = K * np.exp(-19) + (K + 1) * 2.0 ** -23
                assert float(((hard.double() - onehot).abs().amax(0) * clear).max()) <= tol, what
    _lib.poll_kernel_error()


def test_drop_in_aggregate_takes_255_objects(dev, golden):
    """model.aggregate at K in {17, 64, 255} against the reference's outputs (goldens)."""
    from model.aggregate import aggregate_sbg, aggregate_wbg
    g = golden("objects.npz")
    for K in GO.AGG_K:
        p = GO.agg_inputs(K).to(dev)
        for mode, got in (("wbg_hard", aggregate_wbg(p, keep_bg=True, hard=True)),
                          ("wbg_soft", aggregate_wbg(p, keep_bg=True)), ("sbg", aggregate_sbg(p, keep_bg=True))):
            # fp32 on both sides in another order (torch.prod, logf): ~K u relative; the hard logits scale it by 1000
            d = (got.cpu().double() - torch.from_numpy(g[f"agg_K{K}_{mode}"]).double()).abs()
            assert float(d.max()) <= (5e-3 if mode == "wbg_hard" else 1e-4), (K, mode, float(d.max()))
    for bad in (0, 256):
        with pytest.raises(_lib.MivosError, match="1 to 255"):
            aggregate_wbg(torch.rand(bad, 1, 4, 4, device=dev))


# ------------------------------------------------------------------------------------------------ stem gather
@pytest.mark.parametrize("f16", [False, True])
def test_stem_gather_range(dev, f16):
    dt = torch.float16 if f16 else torch.float32
    H, W = 32, 48
    rows = (H // 2 + 2) * (W // 2 + 2)
    kpad = 128 if f16 else 96
    g = torch.Generator().manual_seed(5)
    for K in (5, 16, 40, 255):
        frame = torch.randn((1, 3, H, W), generator=g).to(dev)
        masks = (torch.rand((K, 1, H, W), generator=g) * (torch.rand((K, 1, H, W), generator=g) < 0.3)).to(dev)
        whole = None
        if K <= 16:
            whole = torch.full((K * rows, kpad), SENT, dtype=dt, device=dev)
            ops.stem_gather(frame, masks, whole, s2d=True)
        for k0, n in object_chunks(K) + [(0, K), (K - 1, 1), (1, min(K - 1, 16))]:
            out = torch.full((n * rows, kpad), SENT, dtype=dt, device=dev)
            ops.stem_gather_range(frame, masks, k0, n, out)
            torch.cuda.synchronize()
            if whole is not None:
                assert torch.equal(out, whole[k0 * rows:(k0 + n) * rows]), (K, k0, n)
            ref = stem_reference(frame, masks, k0, n)
            got = out[:, :80].double().cpu()
            err = (got - ref).abs()
            assert bool((err <= stem_tolerance(ref, K, f16)).all()), (K, k0, n, float(err.max()))
            assert bool((out[:, 80:] == 0).all())
    lib = _lib.load()
    before = int(lib.mivos_launch_count())
    out = torch.zeros((rows, kpad), dtype=dt, device=dev)
    for k0, n in ((-1, 1), (0, 0), (4, 2)):
        with pytest.raises(_lib.MivosError, match="stem_gather_s2d_range"):
            ops.stem_gather_range(frame[:, :, :H, :W], masks[:5], k0, n, out)
    assert int(lib.mivos_launch_count()) == before
    _lib.poll_kernel_error()


# ------------------------------------------------------------------------------------------------ networks
@pytest.fixture(scope="module", params=["tf32", "fp16"])
def obj_nets(request, prop_sd, fuse_sd, dev):
    act = torch.float16 if request.param == "fp16" else torch.float32
    nets = {}
    for k in sorted({c[3] for c in GO.CLIPS.values()}):
        net = mivos_b200.PropagationNetwork(top_k=k, act_dtype=act)
        net.load_state_dict(prop_sd, strict=True)
        nets[k] = net.to(dev)
    fuse = mivos_b200.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    return {"nets": nets, "fuse": fuse.to(dev)}


def _close(p, ref, p_max=P_MAX):
    d = (torch.as_tensor(p).cpu() - torch.as_tensor(ref)).abs()
    assert float(d.max()) <= p_max and float(d.mean()) <= P_MEAN, (float(d.max()), float(d.mean()))


def _masks_agree(m, masks_ref, prob_sub, p_max):
    """The u8 masks equal the reference's at every sampled pixel where its two largest probabilities are more than
    2 p_max apart (elsewhere the argmax of K + 1 near-equal probabilities is decided by rounding: with tens of
    overlapping objects and random weights the fused frames are mostly such pixels)."""
    top2 = torch.from_numpy(prob_sub).topk(2, 0).values
    clear = (top2[0] - top2[1]) > 2 * p_max
    ours, ref = torch.from_numpy(m[:, ::GO.SUB, ::GO.SUB]), torch.from_numpy(masks_ref[:, ::GO.SUB, ::GO.SUB])
    print(f"masks: {float(clear.float().mean()):.3f} of the sampled pixels have a clear maximum")
    assert bool((ours == ref)[clear].all()) and float(clear.float().mean()) > 0.05, float(clear.float().mean())


@pytest.mark.parametrize("K", sorted(GO.CLIPS))
def test_clip_matches_reference(dev, obj_nets, golden, K):
    g = golden("objects.npz")
    T, h, w, top_k, mem_freq = GO.CLIPS[K]
    images, mask, mask2 = GO.clip_inputs(K)
    core = mivos_b200.InferenceCore(obj_nets["nets"][top_k], obj_nets["fuse"], images, K, mem_profile=0,
                                    mem_freq=mem_freq, device="cuda:0")
    # 255 objects: the largest difference measured is 0.053 (fp16) / 0.044 (TF32) at a mean of 2e-5
    p_max = P_MAX if K <= 40 else 2 * P_MAX
    m1 = core.interact(mask, 0)
    assert core.bank_trace == [tuple(int(x) for x in r) for r in g[f"clip{K}_trace1"]]
    _close(core.prob[:, :, 0, ::GO.SUB, ::GO.SUB], g[f"clip{K}_prob1_sub"], p_max)
    _masks_agree(m1, g[f"clip{K}_masks1"], g[f"clip{K}_prob1_sub"], p_max)
    core.bank_trace = []
    m2 = core.interact(mask2, T - 1)  # fuse_one_frame on the frames between
    assert core.bank_trace == [tuple(int(x) for x in r) for r in g[f"clip{K}_trace2"]]
    _close(core.prob[:, :, 0, ::GO.SUB, ::GO.SUB], g[f"clip{K}_prob2_sub"], p_max)
    _masks_agree(m2, g[f"clip{K}_masks2"], g[f"clip{K}_prob2_sub"], p_max)
    pm = torch.zeros(K + 1, 1, images.shape[3], images.shape[4])
    pm[K] = 1
    m3 = core.update_mask_only(pm, 1)
    assert (m3[1] == K).all()
    _lib.poll_kernel_error()


def test_graph_replay_equals_eager_at_40_objects(dev, obj_nets, monkeypatch):
    images, mask = Wt.synthetic_clip(6, 112, 176, 40, seed=77)
    res = []
    for on in ("0", "1", "1"):
        monkeypatch.setenv("MIVOS_GRAPH", on)
        core = mivos_b200.InferenceCore(obj_nets["nets"][50], None, images, 40, mem_freq=1, device="cuda:0")
        assert not core._passes_can_overlap(2)  # more than one object chunk: one lane
        m = core.interact(mask, 2)
        res.append((m.copy(), core.prob.clone(), list(core.bank_trace)))
    for m, p, tr in res[1:]:
        assert tr == res[0][2] and torch.equal(p, res[0][1]) and (m == res[0][0]).all()
    _lib.poll_kernel_error()


def test_memorize_and_segment_in_chunks_match_one_batch(dev, obj_nets):
    """The reference-layout memorize at K = 20 runs two chunks of 10 whose keys are the engine's object-range memorize
    of each chunk; segment_with_query takes the 20-object bank; K = 0 and 256 are refused."""
    net = obj_nets["nets"][20]  # a one-frame bank of 4 x 6 slots: top_k 20
    images, mask = Wt.synthetic_clip(2, 64, 96, 20, seed=8)
    frame = images[:, 0].to(dev)
    k16, v16 = net.memorize(frame, mask[1:].to(dev))
    assert k16.shape == (20, 128, 1, 4, 6) and v16.shape == (20, 512, 1, 4, 6)
    # objects 0..9 through the whole-clip gather (K = 10 would change their "others"), compared on the trunk output
    eng = net.engine()
    kv = eng.encode_memory(frame, mask[1:].to(dev), (0, 10))
    assert torch.equal(ops.halo_to_nchw(kv, 10, 4, 6, 128), k16[:10, :, 0])
    qv = net.get_query_values(images[:, 1].to(dev))
    raw = net.segment_with_query(k16, v16, *qv)
    assert raw.shape == (20, 1, 64, 96) and bool(((raw >= 0) & (raw <= 1)).all())
    for bad in (0, 256):
        with pytest.raises(_lib.MivosError, match="1 to 255"):
            mivos_b200.InferenceCore(net, None, images, bad, device="cuda:0")
    _lib.poll_kernel_error()


def test_lockstep_rejects_more_than_16_objects(dev, obj_nets):
    images, _ = Wt.synthetic_clip(3, 64, 96, 17, seed=9)
    cores = [mivos_b200.InferenceCore(obj_nets["nets"][50], None, images, 17, device="cuda:0") for _ in range(2)]
    with pytest.raises(_lib.MivosError, match="at most 16"):
        mivos_b200.LockstepSession(cores)


def test_s2m_controller_takes_20_objects(dev):
    from mivos_b200.s2m import S2MController, S2MNetwork
    net = S2MNetwork(act_dtype=torch.float32).to(dev)
    K, nh, nw = 20, 64, 96
    g = torch.Generator().manual_seed(3)
    image = torch.randn((1, 3, nh, nw), generator=g).to(dev)
    prev = torch.randint(0, K + 1, (1, nh, nw), generator=g).to(dev)
    scr = np.random.default_rng(4).integers(0, K + 2, (nh, nw))
    out = S2MController(net, K, K + 1, device=dev).interact(image, prev, scr)
    ids = np.arange(1, K + 1).reshape(-1, 1, 1)
    x = mivos_b200.s2m.scribble_inputs(image, prev, scr[None] == ids, (scr[None] != ids) & (scr[None] != K + 1))
    for i in (0, 9, 10, 19):  # both chunks (10 + 10), against one object per call (another batch shape, so
        ref = net.forward_sigmoid(x[i:i + 1])  # other convolution plans: the network tests' tolerance)
        assert float((out[i] - ref[0]).abs().max()) <= P_MAX, i
    with pytest.raises(_lib.MivosError, match="1 to 255"):
        S2MController(net, 256, 0)
    _lib.poll_kernel_error()
