"""GPU: the wide top-k memory read (mivos_memory_read_wide, PropagationNetwork(top_k=k) for 64 < k <= 1024) against
float64 on the same fp32 operands: index sets must be IDENTICAL wherever the float64 k-th/(k+1)-th score gap exceeds
TIE_EPS = 1e-5 (closer than that fp32 summation order decides), the read-out within 2e-5 of the output range.  Every
score the read ranks by is the exact fp32 chain of the top-k read, so for k <= 64 both reads give the same bits."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402
from oracle import stm_oracle as O  # noqa: E402  (checker only)

TIE_EPS = 1e-5


def _data(K, cap, hw, seed, dev, sets=1):
    g = torch.Generator().manual_seed(seed)
    bk = torch.randn((K, cap, 128), generator=g).to(dev)
    bv = torch.randn((K, cap, 512), generator=g).to(dev)
    qk = torch.randn((sets, hw, 128) if sets > 1 else (hw, 128), generator=g).to(dev)
    return bk, bv, qk


def _wide(bk, bv, slots, qk, k, ws=None, dyn_slots=None, q_div=0, out=None, **kw):
    if out is None:
        out = torch.zeros((bk.shape[0], qk.shape[-2], 512), device=qk.device)
    out, idx, val = ops.memory_read_wide(bk, bv, slots, qk, k, out, want_topk=True, workspace=ws, dyn_slots=dyn_slots,
                                         q_div=q_div, **kw)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    return out, idx, val


def _f64(bk, bv, slots, qk, k):
    """float64 top-k read on the device: (scores sorted desc [K,hw,k+1], indices [K,hw,k+1], read-out [K,hw,512])."""
    q = (qk / np.float32(math.sqrt(128))).double()
    aff = torch.einsum("ksc,qc->kqs", bk[:, :slots].double(), q)
    kk = min(k + 1, slots)
    vals, ind = torch.topk(aff, kk, dim=2)
    e = torch.exp(vals[..., :k] - vals[..., :1])
    w = e / e.sum(2, keepdim=True)
    K, hw = bk.shape[0], qk.shape[0]
    ref = torch.empty((K, hw, 512), dtype=torch.float64, device=bk.device)
    step = max(1, (1 << 27) // (K * k * 512))  # query chunks of <= 1 GB of gathered rows
    v64 = bv[:, :slots].double()
    for q0 in range(0, hw, step):
        rows = v64[torch.arange(K, device=bk.device)[:, None, None], ind[:, q0:q0 + step, :k]]  # [K,chunk,k,512]
        ref[:, q0:q0 + step] = torch.einsum("kqj,kqjc->kqc", w[:, q0:q0 + step], rows)
    return vals, ind, ref


def _check_f64(bk, bv, slots, qk, k, out, idx, tol=2e-5):
    vals, ind, ref = _f64(bk, bv, slots, qk, k)
    gap = vals[..., k - 1] - vals[..., k] if vals.shape[-1] > k else torch.full(vals.shape[:2], math.inf, device=bk.device)
    same = (idx.long().sort(2)[0] == ind[..., :k].sort(2)[0]).all(2)
    assert bool(same[gap > TIE_EPS].all())
    assert float(same.float().mean()) > 0.99
    ok = same & (gap > TIE_EPS)
    assert float((out.double() - ref)[ok].abs().max()) <= tol * float(ref.abs().max())


@pytest.mark.parametrize("hw", [1, 15, 77, 1620])
@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.parametrize("k", [65, 100, 128, 256, 512, 1024])
def test_matches_f64(dev, k, K, hw):
    slots = max(2 * hw, k + 300)
    bk, bv, qk = _data(K, slots + 64, hw, seed=k * 10 + K + hw, dev=dev)
    out, idx, val = _wide(bk, bv, slots, qk, k)
    _check_f64(bk, bv, slots, qk, k, out, idx)
    # topk_val are the exact scores of topk_idx, descending
    assert bool((val[..., 1:] <= val[..., :-1]).all())


def test_oracle_f64_agrees(dev):
    """The numpy oracle of the top-k read arbitrates the same index sets."""
    K, hw, k, slots = 2, 35, 100, 35 * 6
    bk, bv, qk = _data(K, slots, hw, seed=5, dev=dev)
    out, idx, _ = _wide(bk, bv, slots, qk, k)
    mk = bk.permute(0, 2, 1).cpu().numpy()
    mv = bv.permute(0, 2, 1).cpu().numpy()
    ref, oidx, gap = O.memory_read_f64(mk, mv, qk.t().reshape(1, 128, hw).cpu().numpy(), k)
    same = (np.sort(idx.cpu().numpy().transpose(0, 2, 1), axis=1) == np.sort(oidx, axis=1)).all(1)
    assert same[gap > TIE_EPS].all()
    d = np.abs(out.cpu().numpy().transpose(0, 2, 1) - ref).max(1)
    assert float(d[same & (gap > TIE_EPS)].max()) <= 2e-5 * float(np.abs(ref).max())


def test_nan_past_the_live_count(dev):
    K, hw, k, slots = 2, 77, 256, 1000
    bk, bv, qk = _data(K, slots + 300, hw, seed=7, dev=dev)
    want = _wide(bk, bv, slots, qk, k)
    bk[:, slots:] = float("nan")
    bv[:, slots:] = float("nan")
    got = _wide(bk, bv, slots, qk, k)
    assert all(torch.equal(a, b) for a, b in zip(want, got))
    _check_f64(bk, bv, slots, qk, k, got[0], got[1])


def test_k_equals_live_slots(dev):
    K, hw, k = 2, 15, 300
    bk, bv, qk = _data(K, k, hw, seed=8, dev=dev)
    out, idx, _ = _wide(bk, bv, k, qk, k)
    assert bool((idx.sort(2)[0] == torch.arange(k, device=dev, dtype=torch.int32)).all())
    _check_f64(bk, bv, k, qk, k, out, idx)


@pytest.mark.parametrize("k", [65, 256, 1024])
def test_all_equal_keys_select_the_first_k_slots(dev, k):
    """Every score ties: the band of every query exceeds its candidate region, the exact radix select serves it."""
    K, hw, slots = 2, 77, 5000
    bk, bv, qk = _data(K, slots, hw, seed=9, dev=dev)
    bk[0] = bk[0, 0]
    out, idx, _ = _wide(bk, bv, slots, qk, k)
    assert bool((idx[0] == torch.arange(k, device=dev, dtype=torch.int32)).all())
    ref = bv[0, :k].double().mean(0)
    assert float((out[0].double() - ref).abs().max()) <= 1e-5
    _check_f64(bk[1:], bv[1:], slots, qk, k, out[1:], idx[1:])


@pytest.mark.parametrize("mutate", ["bignorm", "dups", "logits1e3"])
def test_adversarial_keys(dev, mutate):
    K, hw, k, slots = 2, 77, 128, 4000
    bk, bv, qk = _data(K, slots, hw, seed=10, dev=dev)
    if mutate == "bignorm":
        bk[:, 5] *= 1e4
    elif mutate == "dups":  # exact score ties between slot pairs
        bk[:, 1::2] = bk[:, 0::2]
    else:  # scores of +-1e3
        bk *= 1e3 / float((bk[:, :slots] @ (qk.t() / math.sqrt(128))).abs().max())
    out, idx, val = _wide(bk, bv, slots, qk, k)
    assert bool(torch.isfinite(out).all())
    # fp32 scores of magnitude 1e3 carry absolute errors of ~2^-22 * 1e3, which the softmax passes on to the weights
    _check_f64(bk, bv, slots, qk, k, out, idx, tol=2e-5 + (2.0 ** -22 * 1e3 if mutate == "logits1e3" else 0.0))
    if mutate == "dups":  # a tie keeps the lower slot: of each pair at the cut the even one comes first
        i = idx.long()
        s = val
        tie = s[..., 1:] == s[..., :-1]
        assert bool((i[..., 1:][tie] > i[..., :-1][tie]).all())


def test_dyn_slots_graph_replay_and_repeat_are_bit_identical(dev):
    K, hw, k, cap = 2, 1620, 256, 12 * 1620
    bk, bv, qk = _data(K, cap, hw, seed=11, dev=dev)
    lives = (k, hw, 3 * hw + 17, cap)
    want = {live: _wide(bk, bv, live, qk, k) for live in lives}
    again = _wide(bk, bv, lives[2], qk, k)
    assert all(torch.equal(a, b) for a, b in zip(want[lives[2]], again))
    dyn = torch.zeros(4, dtype=torch.int32, device=dev)
    ws = torch.empty(ops.memory_read_wide_workspace_bytes(K, cap, hw, k), dtype=torch.uint8, device=dev)
    out = torch.zeros((K, hw, 512), device=dev)
    idx = torch.zeros((K, hw, k), dtype=torch.int32, device=dev)
    val = torch.zeros((K, hw, k), device=dev)

    def call():
        _lib.check(_lib.lib().mivos_memory_read_wide(ops._ptr(bk), ops._ptr(bv), cap, K, cap, ops._ptr(qk), hw, 0, k,
                                                     ops._ptr(out), 512, 0, 0, 0, ops._ptr(idx), ops._ptr(val),
                                                     ops._ptr(ws), ws.numel(), ops._ptr(dyn), 0, ops._stream()),
                   "mivos_memory_read_wide")

    for live in lives:  # eager with a device-side count
        ops.store_i32(dyn, live)
        call()
        torch.cuda.synchronize()
        assert torch.equal(out, want[live][0]) and torch.equal(idx, want[live][1]) and torch.equal(val, want[live][2])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        call()
        torch.cuda.synchronize()
        with torch.cuda.graph(graph, stream=s):
            call()
    torch.cuda.synchronize()
    for live in reversed(lives):
        ops.store_i32(dyn, live)
        graph.replay()
        torch.cuda.synchronize()
        _lib.poll_kernel_error()
        assert torch.equal(out, want[live][0]) and torch.equal(idx, want[live][1]) and torch.equal(val, want[live][2])


def test_query_sets_match_per_clip_calls(dev):
    C, Kc, hw, k, slots = 3, 2, 77, 200, 900
    bk, bv, qk = _data(C * Kc, slots, hw, seed=12, dev=dev, sets=C)
    out, idx, val = _wide(bk, bv, slots, qk, k, q_div=Kc)
    for c in range(C):
        sl = slice(c * Kc, (c + 1) * Kc)
        o1, i1, v1 = _wide(bk[sl].contiguous(), bv[sl].contiguous(), slots, qk[c].contiguous(), k)
        assert torch.equal(o1, out[sl]) and torch.equal(i1, idx[sl]) and torch.equal(v1, val[sl])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_halo_window(dev, dtype):
    K, h, w, k, slots, C = 2, 7, 11, 100, 800, 640
    bk, bv, qk = _data(K, slots, h * w, seed=13, dev=dev)
    flat = _wide(bk, bv, slots, qk, k)[0]
    fill = torch.full((K, h + 2, w + 2, C), 7.0, dtype=dtype, device=dev)
    halo = fill.clone()
    _wide(bk, bv, slots, qk, k, out=halo, halo_hw=(h, w), out_coff=64)
    inner = halo[:, 1:-1, 1:-1, 64:576].reshape(K, h * w, 512)
    assert torch.equal(inner, flat.to(dtype))
    mask = torch.ones_like(halo, dtype=torch.bool)
    mask[:, 1:-1, 1:-1, 64:576] = False
    assert torch.equal(halo[mask], fill[mask])


@pytest.mark.parametrize("k", [1, 20, 50, 64])
def test_bit_identical_to_topk_read(dev, k):
    K, hw, slots = 3, 1620, 5 * 1620
    bk, bv, qk = _data(K, slots, hw, seed=14 + k, dev=dev)
    out = torch.zeros((K, hw, 512), device=dev)
    o1, i1, v1 = ops.memory_read(bk, bv, slots, qk, k, out.clone(), want_topk=True)
    o2, i2, v2 = _wide(bk, bv, slots, qk, k)
    assert torch.equal(i1, i2) and torch.equal(v1, v2) and torch.equal(o1, o2)


# (K, bank frames, hw) of the cfg-2, cfg-3 and cfg-5 banks (DESIGN.md section 7)
CFG_BANKS = {"cfg2": (1, 20, 1620), "cfg3": (3, 50, 1620), "cfg5": (5, 100, 3600)}


@pytest.mark.parametrize("k", [128, 1024])
@pytest.mark.parametrize("cfg", list(CFG_BANKS))
def test_config_banks_on_sampled_queries(dev, cfg, k):
    K, T, hw = CFG_BANKS[cfg]
    slots = T * hw
    g = torch.Generator(device=dev).manual_seed(15)
    bk = torch.randn((K, slots, 128), generator=g, device=dev)
    bv = torch.randn((K, slots, 512), generator=g, device=dev)
    qk = torch.randn((hw, 128), generator=g, device=dev)
    out, idx, _ = _wide(bk, bv, slots, qk, k)
    pick = torch.randperm(hw, generator=torch.Generator().manual_seed(16))[:64].to(dev)
    _check_f64(bk, bv, slots, qk[pick], k, out[:, pick], idx[:, pick])
    del bk, bv
    torch.cuda.empty_cache()


def test_reference_read_outs(dev, golden):
    """EvalMemoryReader(top_k=k) of the unmodified reference (oracle/gen_golden_wide.py), k in {65, ..., 1024}."""
    from oracle import gen_golden_wide as GW
    g = golden("wide.npz")
    for k in GW.MEMREAD_K:
        for K in GW.MEMREAD_OBJECTS:
            mk, mv, qk = GW.memread_inputs(K, k, GW.memread_seed(K, k))
            _, _, T, h, w = mk.shape
            hw = h * w
            bk = mk.reshape(K, 128, T * hw).transpose(1, 2).contiguous().to(dev)
            bv = mv.reshape(K, 512, T * hw).transpose(1, 2).contiguous().to(dev)
            q = qk.reshape(128, hw).t().contiguous().to(dev)
            out = _wide(bk, bv, T * hw, q, k)[0]
            ref = torch.from_numpy(g[f"memread_k{k}_K{K}_out"]).reshape(K, 512, hw).transpose(1, 2).to(dev)
            assert float((out - ref).abs().max()) <= 2e-5 * float(ref.abs().max()), (k, K)
