"""The dense memory read (mivos_memory_read_dense, PropagationNetwork(top_k=None)) against float64 on the same fp32
operands, with an elementwise bound derived from the kernel's arithmetic (DESIGN.md section 6):

  per query q (live slots s, w = the exact softmax weights, M = max score, D = M - min score):
    eps_q  = 2^-16 * max_s sum_c |q_c k_sc| / sqrt(128)     3xTF32 scores: dropped lo.lo term (2^-22), TF32 rounding
                                                            of the lo parts (2^-21 each), fp32 accumulation over
                                                            48 MMA steps, the fp32 division of q (2^-24)
    tau_q  = 2^-9                                          P rounded to TF32 (2^-11), V read as TF32 (<= 2^-10),
                                                           fp32 accumulation of P.V and of the chunk combine
           + 2 (e^(2 eps_q) - 1)                           a score error d moves a weight by a factor e^(+-2d)
           + 2^-20 (n_steps + 4) (1 + D_q)                 exp / rescale roundings of the online softmax:
                                                           n_steps = tiles per chunk + chunks
    |out - ref|[q, c] <= 2 tau_q * sum_s w_s |v_sc|        (the factor 2: the normalisation sees the same errors)

The bound has teeth: single-TF32 scores, a softmax over the query axis, a missing rescale and a dropped last tile,
emulated in float64 on the host, each exceed it on the test data (test_bound_has_teeth, CPU only)."""
import math

import numpy as np
import pytest
import torch

TILE = 32
Q_TILE = 64


def chunk_tiles(hw: int) -> int:
    """The kernel's partition (memread_dense.cu dense_chunk_tiles): tiles of 32 slots per chunk, a function of hw."""
    qt = -(-hw // Q_TILE)
    return max(8, -(-qt ** 3 // 176))


def _scaled_q(qk32: torch.Tensor) -> torch.Tensor:
    return (qk32.float() / np.float32(math.sqrt(128))).double()  # the fp32 division of the reference


def reference(bk, bv, n, qk):
    """float64 read and bound for one object: bk [cap,128], bv [cap,512] fp32, qk [hw,128] fp32 -> (out, bound)."""
    k, v = bk[:n].double(), bv[:n].double()
    q = _scaled_q(qk)
    s = k @ q.t()                                   # [n, hw]
    w = torch.softmax(s, dim=0)
    out = w.t() @ v                                 # [hw, 512]
    a = (k.abs() @ q.abs().t()).amax(0)             # max_s sum_c |q k|  [hw]
    eps = 2.0 ** -16 * a
    D = s.amax(0) - s.amin(0)
    ct = chunk_tiles(qk.shape[0])
    tiles = -(-n // TILE)
    steps = min(ct, tiles) + -(-tiles // ct)
    tau = 2.0 ** -9 + 2 * torch.expm1(2 * eps) + 2.0 ** -20 * (steps + 4) * (1 + D)
    bound = 2 * tau[:, None] * (w.t() @ v.abs()) + 1e-30
    return out, bound


def ratio(got, out, bound) -> float:
    return float(((got.double() - out).abs() / bound).max())


# ------------------------------------------------------------------ the bound has teeth (host only)
def _tf32(x: torch.Tensor) -> torch.Tensor:
    """Round-to-nearest to TF32 (10 mantissa bits) of fp32 values, as float64."""
    b = x.float().contiguous().view(torch.int32).long()
    b = ((b + 0x1000) & ~0x1FFF) & 0xFFFFFFFF
    return torch.from_numpy(b.to(torch.int64).numpy().astype(np.uint32).view(np.float32)).double()


def _teeth_data(seed=3, n=150, hw=77, sigma=2.0):
    g = torch.Generator().manual_seed(seed)
    bk = torch.randn((n, 128), generator=g) * sigma
    bv = torch.randn((n, 512), generator=g)
    qk = torch.randn((hw, 128), generator=g) * sigma
    return bk, bv, qk


def tf32_midpoint_data(n=150, hw=77, seed=4):
    """Keys whose every element lies just short of a TF32 rounding midpoint, the sign of the rounding error set per
    slot (sigma_s), values correlated with sigma_s: single-pass TF32 scores err by ~2^-11 * sum|q.k| coherently,
    the case a random-data test would not show."""
    g = torch.Generator().manual_seed(seed)
    sig = torch.where(torch.rand((n, 1), generator=g) > 0.5, 1.0, -1.0)
    m = 1.25 + torch.randint(0, 16, (n, 1), generator=g).float() * 2.0 ** -10  # TF32-exact levels in [1, 2)
    bk = (m + sig * 0.99 * 2.0 ** -11).float().expand(n, 128).contiguous()  # TF32 ulp 2^-10: next to a midpoint
    bv = (sig * torch.rand((n, 512), generator=g)).float()
    qk = torch.full((hw, 128), 100.0 / 128 * math.sqrt(128)).float() + 1e-3 * torch.randn((hw, 128), generator=g)
    return bk, bv, qk


def test_bound_has_teeth():
    # 1. single-TF32 scores
    bk, bv, qk = tf32_midpoint_data()
    out, bound = reference(bk, bv, bk.shape[0], qk)
    s1 = _tf32(bk) @ _tf32(_scaled_q(qk).float()).t()
    assert ratio(torch.softmax(s1, 0).t() @ bv.double(), out, bound) > 1.0
    bk, bv, qk = _teeth_data()
    n = bk.shape[0]  # 150 = 4 full tiles of 32 + a partial tile of 22
    out, bound = reference(bk, bv, n, qk)
    k, v, q = bk.double(), bv.double(), _scaled_q(qk)
    s = k @ q.t()
    assert ratio(out, out, bound) == 0.0  # exact arithmetic is inside the bound, the variants are not
    # 2. softmax over the query axis
    assert ratio(torch.softmax(s, 1).t() @ v, out, bound) > 1.0
    # 3. online softmax without the rescale of O (l is rescaled)
    m = torch.full((q.shape[0],), -math.inf, dtype=torch.float64)
    l = torch.zeros_like(m)
    o = torch.zeros((q.shape[0], 512), dtype=torch.float64)
    for t0 in range(0, n, TILE):
        st = s[t0:t0 + TILE]
        m_new = torch.maximum(m, st.amax(0))
        p = torch.exp(st - m_new)
        l = l * torch.exp(m - m_new) + p.sum(0)
        o = o + p.t() @ v[t0:t0 + TILE]
        m = m_new
    assert ratio(o / l[:, None], out, bound) > 1.0
    # 4. the partial last tile dropped
    keep = n // TILE * TILE
    assert ratio(torch.softmax(s[:keep], 0).t() @ v[:keep], out, bound) > 1.0


# ------------------------------------------------------------------ the kernel (GPU)
def _bank(K, cap, n, seed, dev, sigma=1.0):
    g = torch.Generator().manual_seed(seed)
    bk = torch.randn((K, cap, 128), generator=g) * sigma
    bv = torch.randn((K, cap, 512), generator=g)
    bk[:, n:] = float("nan")  # capacity beyond the live count: stale data / NaN must not matter
    bv[:, n:] = float("nan")
    return bk.to(dev), bv.to(dev)


def _check(got, bk, bv, n, qk, q_div=0):
    """got [K, hw, 512] against float64, object by object."""
    K = bk.shape[0]
    worst = 0.0
    for o in range(K):
        qo = qk[o // q_div] if q_div else qk
        out, bound = reference(bk[o].cpu(), bv[o].cpu(), n, qo.cpu())
        r = ratio(got[o].cpu(), out, bound)
        worst = max(worst, r)
    assert worst <= 1.0, worst
    return worst


@pytest.fixture()
def ops():
    from mivos_b200 import _lib, ops
    yield ops
    _lib.poll_kernel_error()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.parametrize("T", [1, 2, 7])
@pytest.mark.parametrize("hw", [1, 15, 77, 1620])
def test_dense_read_within_bound(dev, ops, K, T, hw):
    n = T * hw - 3 if T * hw > 8 else T * hw  # not a multiple of any tile
    cap = n + 37
    bk, bv = _bank(K, cap, n, seed=K * 100 + T * 10 + hw, dev=dev)
    qk = torch.randn((hw, 128), generator=torch.Generator().manual_seed(hw)).to(dev)
    out = torch.full((K, hw, 512), 7.0, device=dev)
    ops.memory_read_dense(bk, bv, n, qk, out)
    assert bool(torch.isfinite(out).all())
    _check(out, bk, bv, n, qk)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["equal_keys", "huge_key", "logits_1e3", "tf32_midpoints"])
def test_dense_read_adversarial(dev, ops, case):
    K, hw, n = 2, 77, 333
    bk, bv = _bank(K, n + 5, n, seed=7, dev=dev)
    g = torch.Generator().manual_seed(8)
    qk = torch.randn((hw, 128), generator=g)
    if case == "tf32_midpoints":  # where single-TF32 scores leave the bound (test_bound_has_teeth)
        mk, mv, qk = tf32_midpoint_data(n, hw)
        bk[:, :n], bv[:, :n] = mk.to(dev), mv.to(dev)
    elif case == "equal_keys":  # uniform weights
        bk[:, :n] = bk[:, :1].clone()
    elif case == "huge_key":  # one-hot weights
        bk[:, 100] = bk[:, 100] * 1e3
        qk = bk[0, 100].cpu().expand(hw, 128) * 1e-3 + qk * 1e-3
    else:  # scores of +-1e3
        base = torch.randn((128,), generator=g)
        qk = base.expand(hw, 128).clone() + 0.01 * qk
        sgn = torch.where(torch.rand((K, n, 1), generator=g) > 0.5, 1.0, -1.0)
        bk[:, :n] = (sgn * base / base.norm() ** 2 * 1e3 * math.sqrt(128)).to(dev)
    qk = qk.contiguous().to(dev)
    out = torch.empty((K, hw, 512), device=dev)
    ops.memory_read_dense(bk, bv, n, qk, out)
    assert bool(torch.isfinite(out).all())
    _check(out, bk, bv, n, qk)
    if case == "huge_key":
        assert float((out[0] - bv[0, 100]).abs().max()) <= 1e-2


@pytest.mark.gpu
def test_dense_read_matches_reference_goldens(dev, ops, golden):
    from oracle.gen_golden_dense import MEMREAD_CASES, memread_inputs
    g = golden("dense.npz")
    for name, (K, T, seed) in MEMREAD_CASES.items():
        mk, mv, qk = memread_inputs(K, T, seed)
        hw, n = 35, T * 35
        bk = mk.reshape(K, 128, n).transpose(1, 2).contiguous().to(dev)
        bv = mv.reshape(K, 512, n).transpose(1, 2).contiguous().to(dev)
        q = qk.reshape(128, hw).t().contiguous().to(dev)
        out = torch.empty((K, hw, 512), device=dev)
        ops.memory_read_dense(bk, bv, n, q, out)
        ref = torch.from_numpy(g[f"memread_{name}_out"]).reshape(K, 512, hw).transpose(1, 2)
        for o in range(K):
            _, bound = reference(bk[o].cpu(), bv[o].cpu(), n, q.cpu())
            assert float(((out[o].cpu().double() - ref[o].double()).abs() / bound).max()) <= 1.0, name


@pytest.mark.gpu
def test_dense_read_bit_identity(dev, ops):
    K, hw, T, C = 2, 77, 9, 3
    n, cap = T * hw - 5, (T + 4) * hw
    bk, bv = _bank(C * K, cap, n, seed=31, dev=dev)
    qk = torch.randn((C, hw, 128), generator=torch.Generator().manual_seed(32)).to(dev)
    eager = torch.empty((C * K, hw, 512), device=dev)
    ops.memory_read_dense(bk, bv, n, qk, eager, q_div=K)
    again = torch.empty_like(eager)
    ops.memory_read_dense(bk, bv, n, qk, again, q_div=K)
    assert torch.equal(eager, again)  # two identical calls
    dyn = torch.tensor([n], dtype=torch.int32, device=dev)
    sized = torch.empty_like(eager)
    ops.memory_read_dense(bk, bv, cap, qk, sized, q_div=K, dyn_slots=dyn)
    assert torch.equal(eager, sized)  # device-side count, host slots = capacity
    for c in range(C):  # C clips in one q_div call == C per-clip calls
        solo = torch.empty((K, hw, 512), device=dev)
        ops.memory_read_dense(bk[c * K:(c + 1) * K], bv[c * K:(c + 1) * K], n, qk[c], solo)
        assert torch.equal(solo, eager[c * K:(c + 1) * K])
    # a captured graph replayed with a changing device-side count == eager reads of each count
    ws = torch.empty(ops.memory_read_dense_workspace_bytes(C * K, cap, hw), dtype=torch.uint8, device=dev)
    out_g = torch.empty_like(eager)
    ops.memory_read_dense(bk, bv, cap, qk, out_g, q_div=K, dyn_slots=dyn, workspace=ws)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.memory_read_dense(bk, bv, cap, qk, out_g, q_div=K, dyn_slots=dyn, workspace=ws)
    for live in (hw, 3 * hw + 1, n, 64):
        dyn.fill_(live)
        graph.replay()
        ref = torch.empty_like(eager)
        ops.memory_read_dense(bk, bv, live, qk, ref, q_div=K)
        torch.cuda.synchronize()
        assert torch.equal(out_g, ref), live


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_dense_read_into_halo_window(dev, ops, dtype):
    K, h, w, T = 2, 5, 7, 3
    hw, n = h * w, T * h * w
    bk, bv = _bank(K, n, n, seed=41, dev=dev)
    qk = torch.randn((hw, 128), generator=torch.Generator().manual_seed(42)).to(dev)
    halo = torch.full((K, h + 2, w + 2, 1024), 3.5, dtype=dtype, device=dev)
    ops.memory_read_dense(bk, bv, n, qk, halo, out_coff=512, halo_hw=(h, w))
    flat = torch.empty((K, hw, 512), device=dev)
    ops.memory_read_dense(bk, bv, n, qk, flat)
    inner = halo[:, 1:-1, 1:-1, 512:].reshape(K, hw, 512)
    assert torch.equal(inner, flat.to(dtype))
    sentinel = halo.clone()
    sentinel[:, 1:-1, 1:-1, 512:] = 3.5
    assert bool((sentinel == 3.5).all())  # nothing outside the window was written


@pytest.mark.gpu
def test_dense_read_rejects_bad_arguments(dev, ops):
    from mivos_b200 import _lib
    bk, bv = _bank(1, 64, 64, seed=1, dev=dev)
    qk = torch.zeros((10, 128), device=dev)
    out = torch.empty((1, 10, 512), device=dev)
    with pytest.raises(_lib.MivosError):
        ops.memory_read_dense(bk, bv, 65, qk, out)  # more live slots than the capacity
    with pytest.raises(_lib.MivosError):
        ops.memory_read_dense(bk, bv, 0, qk, out)


FULL = {"cfg2": (1, 21, 1620), "cfg3": (3, 50, 1620), "cfg5": (5, 100, 3600)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FULL))
def test_dense_read_full_size(dev, ops, name):
    """Bank shapes of BASELINE cfg-2 / cfg-3 / cfg-5 (K objects, T frames, hw at stride 16): finite, and within the
    bound on 64 sampled queries."""
    K, T, hw = FULL[name]
    n = T * hw
    g = torch.Generator(device=dev).manual_seed(5)
    bk = torch.randn((K, n, 128), generator=g, device=dev)
    bv = torch.randn((K, n, 512), generator=g, device=dev)
    qk = torch.randn((hw, 128), generator=g, device=dev)
    out = torch.empty((K, hw, 512), device=dev)
    ops.memory_read_dense(bk, bv, n, qk, out)
    assert bool(torch.isfinite(out).all())
    sel = torch.randperm(hw, generator=torch.Generator().manual_seed(6))[:64].to(dev)
    for o in range(K):
        k, v = bk[o].double(), bv[o].double()
        q = _scaled_q(qk[sel])
        s = k @ q.t()
        wt = torch.softmax(s, dim=0)
        ref = wt.t() @ v
        eps = 2.0 ** -16 * (k.abs() @ q.abs().t()).amax(0)
        D = s.amax(0) - s.amin(0)
        ct, tiles = chunk_tiles(hw), -(-n // TILE)
        steps = min(ct, tiles) + -(-tiles // ct)
        tau = 2.0 ** -9 + 2 * torch.expm1(2 * eps) + 2.0 ** -20 * (steps + 4) * (1 + D)
        bound = 2 * tau[:, None] * (wt.t() @ v.abs()) + 1e-30
        assert float(((out[o, sel].double() - ref).abs() / bound).max()) <= 1.0, (name, o)
