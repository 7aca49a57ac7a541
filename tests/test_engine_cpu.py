"""CPU: the HOST side of the propagation engines (mivos_b200/engine.py: weight packing, BatchNorm
folding, the fused key|value projection, stride-2 gathers, concat windows, the decoder's precomputed
skip paths and their broadcast over objects, the bank layout) driven over a PyTorch emulation of the
C-ABI operators (tests/abi_emulator.py, written from include/mivos_b200.h) and compared with the
vectors the UNMODIFIED reference produced (tests/golden/ops_lowres.npz).  The kernels themselves are
checked on the GPU (tests/test_gpu_*.py).  Tolerance: packed weights are rounded to TF32."""
import pytest
import torch

import abi_emulator
from mivos_b200 import engine, ops

TOL = 4e-3


def _close(a, b, tol=TOL):
    b = torch.as_tensor(b)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = float((a - b).abs().max()) / float(b.abs().max())
    assert err <= tol, err


@pytest.fixture()
def eng(prop_sd, monkeypatch):
    abi_emulator.install(monkeypatch, ops)
    return engine.PropagationEngine(prop_sd, "cpu", top_k=20, act_dtype=torch.float32)


def test_query_pass_and_memorize_host_graph(eng, golden):
    g = golden("ops_lowres.npz")
    frame, mask = torch.from_numpy(g["frame"]), torch.from_numpy(g["mask"])
    qs = eng.encode_query(frame, None, keep_features=True)
    nchw = lambda t, c, s, coff=0: ops.halo_to_nchw(t, 1, 96 // s, 128 // s, c, coff=coff)  # noqa: E731
    _close(nchw(qs.f16, 1024, 16), g["f16"])
    _close(nchw(qs.f8, 512, 8)[:, ::4], g["f8"])
    _close(nchw(qs.f4, 256, 4)[:, ::8], g["f4"])
    _close(nchw(qs.kv, 128, 16), g["k16"])
    _close(nchw(qs.kv, 512, 16, coff=128), g["v16"])
    assert torch.equal(qs.qk, qs.kv[0, 1:-1, 1:-1, :128].reshape(-1, 128))  # pixel-major keys for the read
    kv = eng.encode_memory(frame, mask[1:])
    _close(ops.halo_to_nchw(kv, 2, 6, 8, 128), g["mem_k"][:, :, 0])
    _close(ops.halo_to_nchw(kv, 2, 6, 8, 512, coff=128), g["mem_v"][:, :, 0])


def test_batched_query_pass_equals_single_frames(eng, golden):
    g = golden("ops_lowres.npz")
    frames = torch.cat([torch.from_numpy(g["frame"]), torch.from_numpy(g["frame3"])], 0)
    states, batch = eng.new_query_states(96, 128, 2)
    eng.encode_query_batch(frames, batch)
    kv_b, s8_b, s4_b = batch.kv.clone(), batch.s8.clone(), batch.s4.clone()
    for i in range(2):
        one = eng.encode_query(frames[i:i + 1])
        assert float((kv_b[i:i + 1] - one.kv).abs().max()) <= 1e-5
        assert float((s8_b[i:i + 1] - one.s8).abs().max()) <= 1e-5 and float((s4_b[i:i + 1] - one.s4).abs().max()) <= 1e-5
        assert states[i].kv.data_ptr() == batch.kv[i:i + 1].data_ptr()  # state i is a view of the batch


def test_segment_host_graph(eng, golden):
    """Bank from the reference's keys/values, query state from our own query pass: memory read +
    decoder tail (precomputed skip paths, broadcast over the two objects) + x4 resize + sigmoid +
    aggregation against the reference's segment_with_query / aggregate_wbg outputs."""
    g = golden("ops_lowres.npz")
    keys, values = torch.from_numpy(g["keys"]), torch.from_numpy(g["values"])
    K, _, T, h, w = keys.shape
    bank_k, bank_v = torch.zeros((K, T * h * w + 7, 128)), torch.zeros((K, T * h * w + 7, 512))
    ops.bank_from_nchw(keys, values, bank_k, bank_v)
    qs = eng.encode_query(torch.from_numpy(g["frame3"]))
    raw, prob = eng.segment(bank_k, bank_v, T * h * w, qs, K, want_raw=True)
    ref = torch.from_numpy(g["seg"])
    assert float((raw - ref).abs().max()) <= 3e-2 and float((raw - ref).abs().mean()) <= 1e-3
    assert float((prob - torch.from_numpy(g["agg"])).abs().max()) <= 3e-2
    assert float((prob.sum(0) - 1).abs().max()) <= 1e-5
    # the decoder input is [memory read-out (512) | query value (512)] per object (prop_net.py:178-179)
    cat = eng.ws.halo("cat", K, h, w, 1024)
    assert torch.equal(cat[1, 1:-1, 1:-1, 512:], qs.kv[0, 1:-1, 1:-1, 128:])
    # and with the reference's own query key the read-out of object 0 is the reference's (this pins the
    # emulated operator itself; ours above used the key of our TF32-weight query pass)
    rd = torch.zeros((1, h * w, 512))
    ops.memory_read(bank_k[0:1], bank_v[0:1], T * h * w, torch.from_numpy(g["qk3"]).reshape(128, h * w).t().contiguous(), 20, rd)
    _close(rd.reshape(1, h, w, 512).permute(0, 3, 1, 2), g["read"], 1e-5)


def test_fusion_host_graph(fuse_sd, golden, monkeypatch):
    abi_emulator.install(monkeypatch, ops)
    g = golden("ops_lowres.npz")
    fe = engine.FusionEngine(fuse_sd, "cpu")
    t = lambda k: torch.from_numpy(g[k])  # noqa: E731
    nc, nr = (float(v) for v in g["dist"].reshape(-1))
    lg, H, W = fe.forward_logit_halo(t("frame3"), t("seg")[0:1], t("agg")[1:2], t("attn"), nc, nr)
    _close(ops.halo_to_nchw(lg, 1, H, W, 1), g["fuse"])


def test_segment_and_memorize_of_c_clips_equal_per_clip_calls(eng, golden):
    """segment / encode_memory at C = 3 (C clips advanced as one batch of C*K maps, per-clip memory read / skip
    broadcast / stem gather / aggregation as groups) equal the same methods at C = 1 per clip."""
    g = golden("ops_lowres.npz")
    keys, values = torch.from_numpy(g["keys"]), torch.from_numpy(g["values"])
    K, _, T, h, w = keys.shape
    C, slots = 3, T * h * w
    gen = torch.Generator().manual_seed(3)
    frames = torch.cat([torch.from_numpy(g["frame3"]), torch.from_numpy(g["frame"]), torch.randn((1, 3, 96, 128), generator=gen)], 0)
    bank_k, bank_v = torch.zeros((C * K, slots + 5, 128)), torch.zeros((C * K, slots + 5, 512))
    for c in range(C):  # every clip its own bank: permute / perturb the reference's
        kc = keys.roll(c, 0) + 0.05 * c * torch.randn(keys.shape, generator=gen)
        vc = values.roll(c, 0) + 0.05 * c * torch.randn(values.shape, generator=gen)
        ops.bank_from_nchw(kc, vc, bank_k[c * K:(c + 1) * K], bank_v[c * K:(c + 1) * K])
    states, batch = eng.new_query_states(96, 128, C)
    eng.encode_query_batch(frames, batch)
    _, prob_multi = eng.segment(bank_k, bank_v, slots, batch, K, C, prob_out=torch.zeros((C, K + 1, 1, 96, 128)))
    for c in range(C):
        _, prob = eng.segment(bank_k[c * K:(c + 1) * K], bank_v[c * K:(c + 1) * K], slots, states[c], K)
        assert float((prob_multi[c] - prob).abs().max()) <= 1e-5, c
    assert float((prob_multi[0] - torch.from_numpy(g["agg"])).abs().max()) <= 3e-2  # clip 0 is the golden case
    # memorize: clip c's masks are its own probabilities
    masks = prob_multi[:, 1:].contiguous()
    kv_multi = eng.encode_memory(frames, masks).clone()
    for c in range(C):
        kv = eng.encode_memory(frames[c:c + 1], masks[c])
        assert float((kv_multi[c * K:(c + 1) * K] - kv).abs().max()) <= 1e-4, c


def test_workspace_buffers_are_never_replaced():
    """Captured CUDA graphs keep raw pointers into workspace buffers: a request that does not fit an
    existing scratch buffer must get ANOTHER buffer (size classes), never a grown replacement."""
    ws = engine.Workspace("cpu", torch.float32)
    a = ws.raw("scratch", 1000)
    assert ws.raw("scratch", 900) is a and ws.raw("scratch", 1 << 20) is a and a.numel() == 1 << 20
    b = ws.raw("scratch", (1 << 20) + 1)
    assert b is not a and b.numel() == 1 << 21 and ws.raw("scratch", 1000) is a  # the small class is still served by `a`
    h1 = ws.halo("x", 1, 4, 6, 8)
    assert ws.halo("x", 1, 4, 6, 8) is h1 and ws.halo("x", 2, 4, 6, 8) is not h1
    assert h1.shape == (1, 6, 8, 8) and float(h1.abs().max()) == 0
    assert ws.bytes() >= a.numel() + b.numel()
