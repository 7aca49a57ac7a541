"""CPU: host-side logic of the drop-in surface (no kernels are launched)."""
import pytest
import torch

import mivos_b200
from mivos_b200 import arch, ops, tensor_util
from mivos_b200._lib import MivosError


def test_state_dict_surface_matches_reference_format(prop_sd, fuse_sd):
    net = mivos_b200.PropagationNetwork(top_k=20)
    sd = net.state_dict()
    assert list(sd.keys()) != [] and set(sd.keys()) == set(prop_sd.keys()) and len(sd) == 597
    for k, v in prop_sd.items():
        assert tuple(sd[k].shape) == tuple(v.shape), k
    assert net.load_state_dict(prop_sd, strict=True).missing_keys == []
    assert net.memory.top_k == 20 and net.top_k == 20
    f = mivos_b200.FusionNet()
    assert set(f.state_dict().keys()) == set(fuse_sd.keys())
    f.load_state_dict(fuse_sd, strict=True)
    # AttentionReadNetwork-style partial load (fusion_model.py:187) keeps working: sub-module names are ABI
    part = {k: v for k, v in prop_sd.items() if k.split(".")[0] in ("mask_rgb_encoder", "rgb_encoder", "kv_m_f16", "kv_q_f16")}
    assert len(part) > 500


def test_reference_import_paths():
    from inference_core import InferenceCore
    from model.aggregate import aggregate_sbg, aggregate_wbg
    from model.fusion_net import FusionNet
    from model.propagation.prop_net import PropagationNetwork
    from util.tensor_util import pad_divide_by, unpad
    assert InferenceCore is mivos_b200.InferenceCore and PropagationNetwork is mivos_b200.PropagationNetwork
    assert FusionNet is mivos_b200.FusionNet and callable(aggregate_wbg) and callable(aggregate_sbg)
    assert callable(pad_divide_by) and callable(unpad)


def test_no_cpu_fallback():
    net = mivos_b200.PropagationNetwork()
    with pytest.raises(MivosError):
        net.get_query_values(torch.zeros(1, 3, 32, 32))
    with pytest.raises(MivosError):
        mivos_b200.InferenceCore(net, None, torch.zeros(1, 2, 3, 32, 32), 1, device="cpu")
    with pytest.raises(MivosError):
        ops.aggregate_wbg(torch.zeros(1, 1, 4, 4))


@pytest.mark.parametrize("h,w,exp", [(480, 854, (5, 5, 0, 0)), (480, 864, (0, 0, 0, 0)), (5, 7, (4, 5, 5, 6)), (720, 1280, (0, 0, 0, 0))])
def test_pad_amounts_match_reference_formula(h, w, exp):
    assert tensor_util.pad_amounts(h, w, 16) == exp
    x = torch.zeros(1, 1, h, w)
    y, pad = tensor_util.pad_divide_by(x, 16)  # CPU tensors are staged with F.pad (host plumbing)
    assert pad == exp and y.shape[-2] % 16 == 0 and y.shape[-1] % 16 == 0
    assert tensor_util.unpad(y, pad).shape == x.shape


def test_pack_conv_folds_batchnorm_and_rounds_to_tf32():
    torch.manual_seed(0)
    w = torch.randn(8, 5, 3, 3)
    b = torch.randn(8)
    bn = (torch.rand(8) + 0.5, torch.randn(8), torch.randn(8), torch.rand(8) + 0.5, 1e-5)
    pc = ops.pack_conv(w, b, bn=bn, device="cpu")
    assert pc.taps == 9 and pc.cin_pad == 32 and pc.cout_pad == 32 and pc.weight.shape == (9, 32, 32)
    x = torch.randn(1, 5, 6, 6)
    ref = torch.nn.functional.batch_norm(torch.nn.functional.conv2d(x, w, b, padding=1), bn[2], bn[3], bn[0], bn[1], False, 0.0, 1e-5)
    wfold = pc.weight[:, :8, :5].reshape(3, 3, 8, 5).permute(2, 3, 0, 1)
    got = torch.nn.functional.conv2d(x, wfold, pc.bias[:8], padding=1)
    assert float((got - ref).abs().max()) < 5e-3 * float(ref.abs().max())  # only TF32 rounding of the weights
    assert (pc.weight.view(torch.int32) & 0x1FFF).abs().max() == 0  # low 13 mantissa bits cleared
    pc7 = ops.pack_conv(torch.randn(64, 5, 7, 7), None, stride=2, im2col=True, device="cpu")
    assert pc7.taps == 1 and pc7.cin_pad == 256 and pc7.cin == 5


def test_arch_tables():
    ents = arch.propagation_entries()
    convs = [e for e in ents if e[0] == "conv"]
    bns = [e for e in ents if e[0] == "bn"]
    assert len(convs) == 2 * (1 + 13 * 3 + 3) + 4 + 15 == 105 and len(bns) == 2 * (1 + 13 * 3 + 3) == 86
    assert len(arch.fusion_entries()) == 6


def test_synth_generator_equals_oracle_generator(prop_sd, fuse_sd):
    """Two independently written architecture tables (mivos_b200/arch.py, oracle/weights.py) + the
    same RNG recipe must give identical checkpoints and clips."""
    from mivos_b200 import synth
    from oracle import weights as Wt
    a = synth.make_prop_state_dict(1234)
    assert list(a.keys()) == list(prop_sd.keys()) and all(torch.equal(a[k], prop_sd[k]) for k in a)
    b = synth.make_fusion_state_dict(4321)
    assert all(torch.equal(b[k], fuse_sd[k]) for k in b)
    i1, m1 = synth.synthetic_clip(3, 64, 96, 2, seed=9)
    i2, m2 = Wt.synthetic_clip(3, 64, 96, 2, seed=9)
    assert torch.equal(i1, i2) and torch.equal(m1, m2)


def test_conv_tile_plan_matches_the_on_device_sweep():
    """mivos_conv_plan is the host-side cost model of mivos_conv_gemm (no device needed): on the
    shapes of the cfg-2 frame, planned for the 132 SMs of an H100, it must pick a tile width that the on-device sweep
    measured as best or within 5 % of it, and only split K where a workspace is attached."""
    import ctypes as C
    from mivos_b200 import _lib
    lib = _lib.load()

    def plan(n, h, w, cin, cout, ks, res=False, ws=False, f16=True):
        a = _lib.ConvArgs()
        a.n, a.h, a.w = n, h, w
        a.taps = 9 if ks == 3 else 1
        q = 64 if f16 else 32
        a.cin_pad = (cin + q - 1) // q * q
        a.cout, a.cout_pad = cout, (cout + 31) // 32 * 32
        a.in_f16 = a.out_f16 = int(f16)
        a.residual = 16 if res else None   # never dereferenced by the planner
        if ws:
            a.splitk_ws, a.splitk_ws_bytes = 256, 48 << 20
        bn, sp = C.c_int(0), C.c_int(0)
        assert lib.mivos_conv_plan(C.byref(a), 132, C.byref(bn), C.byref(sp)) == 0, lib.mivos_last_error()
        return bn.value, sp.value

    # (shape) -> admissible tile widths: within 5 % of the best of tools/tile_sweep.py on an H100 80GB HBM3 (fp16 maps,
    # graph-replayed; times in us per launch)
    assert plan(1, 120, 216, 256, 256, 3)[0] in (256,)          # 198.4 @32, 115.2 @64, 81.5 @128, 58.8 @256
    assert plan(1, 60, 108, 512, 512, 3)[0] in (256,)          # 196.9 @32, 123.1 @64, 75.0 @128, 52.3 @256
    assert plan(1, 60, 108, 512, 256, 3)[0] in (128,)          # 112.4 @32, 62.6 @64, 38.1 @128, 50.6 @256
    assert plan(1, 30, 54, 256, 256, 3)[0] in (32,)           # 15.6 @32, 17.0 @64, 20.2 @128, 28.1 @256
    assert plan(1, 30, 54, 1024, 256, 1)[0] in (32,)           # 8.2 @32, 9.1 @64, 11.1 @128, 16.2 @256
    assert plan(1, 30, 54, 256, 1024, 1, res=True)[0] in (128,)          # 21.9 @32, 12.0 @64, 9.7 @128, 16.5 @256
    assert plan(1, 120, 216, 64, 256, 1, res=True)[0] in (128, 256)      # 72.0 @32, 37.5 @64, 35.4 @128, 33.9 @256
    assert plan(8, 30, 54, 256, 256, 3)[0] in (256,)          # 106.3 @32, 65.8 @64, 41.0 @128, 29.6 @256
    assert plan(8, 120, 216, 64, 256, 1, res=True)[0] in (256,)          # 753.9 @32, 392.4 @64, 339.2 @128, 310.4 @256
    assert plan(4, 120, 216, 64, 256, 1, res=True)[0] in (128, 256)      # 366.6 @32, 195.2 @64, 171.6 @128, 164.2 @256
    assert plan(4, 60, 108, 128, 512, 1, res=True)[0] in (128, 256)      # 181.7 @32, 100.9 @64, 93.2 @128, 97.2 @256
    assert plan(8, 30, 54, 256, 1024, 1, res=True)[0] in (128, 256)      # 216.9 @32, 120.0 @64, 102.8 @128, 105.3 @256
    assert plan(4, 120, 216, 256, 256, 3, res=True)[0] in (256,)          # 959.1 @32, 526.4 @64, 369.3 @128, 318.8 @256
    assert plan(8, 60, 108, 512, 128, 1)[0] in (128,)          # 97.0 @32, 56.8 @64, 40.1 @128
    # split-K: only with a workspace, and only for the K >= 9 x 512 layers of the small maps
    assert plan(1, 30, 54, 1024, 512, 3, ws=False)[1] == 1
    bn, sp = plan(1, 30, 54, 1024, 512, 3, ws=True)
    assert bn >= 128 and sp >= 2
    assert plan(1, 30, 54, 256, 256, 3, ws=True)[1] == 1
    assert plan(1, 120, 216, 256, 256, 3, ws=True)[1] == 1
    assert plan(8, 30, 54, 1024, 256, 1, ws=True)[1] == 1


def test_attention_read_network_checkpoint_surface(prop_sd):
    """model/attn_network.py:30-41 + fusion_model.py:187: same sub-module names as the propagation
    network minus the decoder, so a propagation checkpoint loads with strict=False and nothing is
    missing; a CPU instance refuses to run (no CPU path)."""
    import mivos_b200
    from mivos_b200._lib import MivosError
    net = mivos_b200.AttentionReadNetwork()
    keys = set(net.state_dict())
    assert keys == {k for k in prop_sd if not k.startswith("decoder.")} and len(keys) == 567
    r = net.load_state_dict(prop_sd, strict=False)
    assert not r.missing_keys and all(k.startswith("decoder.") for k in r.unexpected_keys)
    assert all(not p.requires_grad for p in net.parameters())  # attn_network.py:40-41
    z = torch.zeros(1, 1, 32, 32)
    with pytest.raises(MivosError):
        net(torch.zeros(1, 3, 32, 32), z, z, z, z, torch.zeros(1, 3, 32, 32))


def test_pass_plan_equals_oracle_bank_trace(prop_sd, fuse_sd):
    """schedule.plan_pass (the bookkeeping InferenceCore.do_pass and the lock-step driver execute)
    against the trace of the oracle's restatement of inference_core.py:122-200, over three
    interactions (forward + backward passes, passes bounded by other interactions -> fusion)."""
    import torch
    from mivos_b200 import schedule
    from oracle import stm_oracle as O, weights as Wt
    t, mem_freq = 10, 2
    images, mask = Wt.synthetic_clip(t, 64, 96, 1, seed=2)  # 24 slots per bank frame >= top_k
    oc = O.OracleInferenceCore(prop_sd, fuse_sd, images, 1, mem_freq=mem_freq, top_k=20)
    interacted, num_certain = set(), 0
    for idx in (3, 8, 0):
        oc.bank_trace = []
        oc.interact(mask, idx)
        interacted.add(idx)
        num_certain += 1
        got = []
        for forward in (True, False):
            plan = schedule.plan_pass(t, interacted, idx, forward, mem_freq, num_certain)
            got += [(f.ti, f.visible) for f in plan.frames]
            assert all(f.memorize for f in plan.frames[:-1]) and (not plan.frames or not plan.frames[-1].memorize)
            assert all(f.visible <= plan.total_m and f.m_front < plan.total_m for f in plan.frames if f.memorize)
            assert plan.fuse == (plan.closest_ti not in (-1, t))
            assert schedule.bank_capacity_frames(t, mem_freq, num_certain, plan.total_m) >= plan.total_m
        assert got == oc.bank_trace, (idx, got, oc.bank_trace)


def test_pass_plan_cfg2_shape():
    """BASELINE configs[1]: 101-frame clip, mem_freq 5, interaction on frame 0: the bank grows 1 -> 20
    committed frames + the interacted one (+ the temporary slot), the last frame is never memorised."""
    from mivos_b200 import schedule
    plan = schedule.plan_pass(101, {0}, 0, True, 5, 1)
    assert (plan.closest_ti, plan.total_m, plan.fuse, len(plan.frames)) == (101, 22, False, 100)  # 21 + the temporary slot
    assert plan.frames[0] == schedule.FramePlan(1, 1, 1, True) and plan.frames[1].visible == 2
    assert plan.frames[-1] == schedule.FramePlan(100, 21, 20, False)
    assert max(f.visible for f in plan.frames) == 21
    back = schedule.plan_pass(101, {0}, 0, False, 5, 1)
    assert back.frames == [] and back.closest_ti == -1


def test_second_interaction_mask_recipe_matches_the_golden_generator():
    from mivos_b200 import synth
    from oracle import gen_golden_full as G
    a = synth.second_interaction_mask(2, 64, 96, seed=77)
    b = G.second_mask(2, 64, 96, 77)
    assert torch.equal(a, b) and float(a.sum(0).min()) == 1.0 and float(a.sum(0).max()) == 1.0


def test_aggregate_wbg_channel_matches_the_reference_formula():
    """model/aggregate.py:39-54 (training-time twin, torch-only here): logits + softmax over dim 1."""
    from mivos_b200.aggregate import aggregate_wbg_channel
    import model.aggregate as shim
    assert shim.aggregate_wbg_channel is aggregate_wbg_channel
    g = torch.Generator().manual_seed(3)
    prob = torch.rand((2, 3, 8, 8), generator=g)
    new = torch.cat([torch.prod(1 - prob, dim=1, keepdim=True), prob], 1).clamp(1e-7, 1 - 1e-7)
    logits = torch.log(new / (1 - new))
    lg, sm = aggregate_wbg_channel(prob, keep_bg=True)
    assert torch.equal(lg, logits) and torch.equal(sm, torch.softmax(logits, dim=1))
    lg2, sm2 = aggregate_wbg_channel(prob, keep_bg=False, hard=True)
    assert torch.equal(lg2, logits * 1000) and sm2.shape == (2, 3, 8, 8)
