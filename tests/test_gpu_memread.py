"""GPU: the fused space-time memory read (affinity -> top-k -> softmax -> value read-out) through
the C ABI, both candidate generators (exact CUDA-core and tensor-core), against
  * the committed golden vectors produced by the reference's EvalMemoryReader,
  * the float64 oracle (index sets must be IDENTICAL wherever the oracle's k-th/(k+1)-th score gap
    exceeds TIE_EPS = 1e-5; closer than that fp32 summation order decides, also inside the
    reference itself — SURVEY.md §7 hard parts),
  * each other: the two generators must agree BIT FOR BIT (final scores are always re-computed with
    the same fp32 FMA chain, the TF32 tensor-core scores only pre-select),
  * size-independent properties at BASELINE.json's full cfg-2 size.
Read-out tolerance vs the fp32 reference result: 2e-5 of the output range (fp32 round-off of a
k-term weighted sum)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402
from oracle import stm_oracle as O  # noqa: E402  (checker only)

TIE_EPS = 1e-5
ALGOS = [ops.MEMREAD_EXACT_SIMT, ops.MEMREAD_TCGEN05]


def _bank(mk, mv, dev, extra=0):
    K, _, T, h, w = mk.shape
    bk = torch.zeros((K, T * h * w + extra, 128), device=dev)
    bv = torch.zeros((K, T * h * w + extra, 512), device=dev)
    ops.bank_from_nchw(mk.contiguous(), mv.contiguous(), bk, bv)
    return bk, bv


def _read(bk, bv, slots, qpm, k, algo, ws=None):
    out = torch.zeros((bk.shape[0], qpm.shape[0], 512), device=qpm.device)
    out, idx, val = ops.memory_read(bk, bv, slots, qpm, k, out, algo=algo, want_topk=True, workspace=ws)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    return out, idx, val


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("k", [20, 50])
def test_golden_vectors(dev, golden, algo, k):
    g = golden("memread.npz")
    mk, mv, qk = (torch.from_numpy(g[n]).to(dev) for n in ("mk", "mv", "qk"))
    K, _, T, h, w = mk.shape
    hw = h * w
    bk, bv = _bank(mk, mv, dev)
    out, idx, _ = _read(bk, bv, T * hw, qk.reshape(128, hw).t().contiguous(), k, algo)
    ref = torch.from_numpy(g[f"out{k}"]).reshape(K, 512, hw).transpose(1, 2).to(dev)
    assert float((out - ref).abs().max()) <= 2e-5 * float(ref.abs().max())
    _, oidx, gap = O.memory_read_f64(g["mk"], g["mv"], g["qk"], k)
    ours = np.sort(idx.cpu().numpy().transpose(0, 2, 1), axis=1)
    same = (ours == np.sort(oidx, axis=1)).all(1)
    assert same[gap > TIE_EPS].all() and same.mean() > 0.99


@pytest.mark.parametrize("K,T,h,w,k,extra,mutate", [
    (1, 1, 30, 54, 20, 0, None),       # single-frame bank (first propagated frame)
    (1, 3, 30, 54, 20, 0, None),
    (2, 5, 30, 54, 50, 0, None),
    (2, 9, 7, 9, 20, 5, None),         # hw=63 (< one query tile), ragged slot count
    (1, 13, 10, 20, 50, 77, None),
    (1, 1, 6, 8, 20, 0, None),         # 48 slots: fewer slots than one tile
    (1, 4, 30, 54, 20, 0, "dups"),     # every key duplicated: exact score ties
    (2, 3, 30, 54, 20, 0, "equal"),    # object 0: all keys equal -> candidate overflow -> exact fallback
    (1, 4, 30, 54, 20, 0, "bignorm"),  # one huge key blows the TF32 margin up -> fallback
])
def test_generators_agree_bit_for_bit_and_match_f64(dev, K, T, h, w, k, extra, mutate):
    g = torch.Generator().manual_seed(K * 1000 + T * 10 + k)
    hw = h * w
    slots = T * hw + extra
    bk = torch.randn((K, slots + 300, 128), generator=g).to(dev)
    bv = torch.randn((K, slots + 300, 512), generator=g).to(dev)
    qk = torch.randn((hw, 128), generator=g).to(dev)
    if mutate == "dups":
        bk[:, 1:slots:2] = bk[:, 0:slots - 1:2]
    elif mutate == "equal":
        bk[0, :] = bk[0, 0]
    elif mutate == "bignorm":
        bk[:, 5] *= 50.0
    o1, i1, v1 = _read(bk, bv, slots, qk, k, ops.MEMREAD_EXACT_SIMT)
    o2, i2, v2 = _read(bk, bv, slots, qk, k, ops.MEMREAD_TCGEN05)
    assert torch.equal(i1, i2) and torch.equal(v1, v2) and torch.equal(o1, o2)
    # float64 check of the selection and the read-out
    aff = torch.einsum("ksc,qc->ksq", bk[:, :slots].double(), (qk / (128 ** 0.5)).double())
    vals, ind = torch.topk(aff, k + 1, dim=1)
    gap = (vals[:, k - 1] - vals[:, k])
    same = (i1.long().transpose(1, 2).sort(1)[0] == ind[:, :k].sort(1)[0]).all(1)
    assert bool(same[gap > TIE_EPS].all())
    if mutate is None:
        e = torch.exp(vals[:, :k] - vals[:, :1])
        wgt = e / e.sum(1, keepdim=True)
        ref = torch.einsum("kjq,kjqc->kqc", wgt, bv[:, :slots].double()[torch.arange(K)[:, None, None], ind[:, :k]])
        ok = same & (gap > TIE_EPS)
        assert float((o1.double() - ref)[ok].abs().max()) <= 2e-5 * float(ref.abs().max())


def test_cfg2_full_size_properties(dev):
    """BASELINE configs[1] steady state: 1 object, 20-frame bank, 480p (hw=1620), top-k 20."""
    g = torch.Generator().manual_seed(2)
    K, T, hw, k = 1, 20, 1620, 20
    slots = T * hw
    bk = torch.randn((K, slots, 128), generator=g).to(dev)
    bv = torch.randn((K, slots, 512), generator=g).to(dev)
    qk = torch.randn((hw, 128), generator=g).to(dev)
    o_tc, i_tc, v_tc = _read(bk, bv, slots, qk, k, ops.MEMREAD_TCGEN05)
    o_ex, i_ex, v_ex = _read(bk, bv, slots, qk, k, ops.MEMREAD_EXACT_SIMT)
    assert torch.equal(i_tc, i_ex) and torch.equal(o_tc, o_ex)
    # scores come back sorted (descending) and indices are unique per query
    assert bool((v_tc[..., :-1] >= v_tc[..., 1:]).all())
    assert int(i_tc.sort(-1)[0].diff(dim=-1).eq(0).sum()) == 0
    # linearity in the values (exact for a power-of-two scale) and convexity of the weights
    o2, _, _ = _read(bk, bv * 2.0, slots, qk, k, ops.MEMREAD_TCGEN05)
    assert torch.equal(o2, o_tc * 2.0)
    ones, _, _ = _read(bk, torch.ones_like(bv), slots, qk, k, ops.MEMREAD_TCGEN05)
    assert float((ones - 1).abs().max()) <= 1e-6
    # permuting the bank slots permutes the selected indices and leaves the read-out unchanged
    # up to the fp32 order of the k-term sum
    perm = torch.randperm(slots, generator=g).to(dev)
    o3, i3, v3 = _read(bk[:, perm].contiguous(), bv[:, perm].contiguous(), slots, qk, k, ops.MEMREAD_TCGEN05)
    assert torch.equal(v3, v_tc)
    assert torch.equal(perm[i3.long()].sort(-1)[0], i_tc.long().sort(-1)[0])
    assert float((o3 - o_tc).abs().max()) <= 1e-5 * float(o_tc.abs().max())


@pytest.mark.parametrize("name,K,T,hw,k", [
    ("cfg3", 3, 50, 1620, 50),    # BASELINE configs[2]: 480p, 3 objects, 50-frame bank, top-k 50
    ("cfg5", 5, 100, 3600, 50),   # BASELINE configs[4]: 720p, 5 objects, 100-frame bank (4.6 GB of bank)
])
def test_full_size_configs_properties(dev, name, K, T, hw, k):
    """Full-size memory banks of the larger BASELINE configurations: the tensor-core candidate path and
    the exact SIMT path must select the same slots and produce the same read-out bit for bit;
    size-independent properties: sorted scores, unique indices, convex weights."""
    g = torch.Generator(device=dev).manual_seed(K * 100 + T)
    slots = T * hw
    bk = torch.randn((K, slots, 128), generator=g, device=dev)
    bv = torch.randn((K, slots, 512), generator=g, device=dev)
    qk = torch.randn((hw, 128), generator=g, device=dev)
    o_tc, i_tc, v_tc = _read(bk, bv, slots, qk, k, ops.MEMREAD_TCGEN05)
    o_ex, i_ex, v_ex = _read(bk, bv, slots, qk, k, ops.MEMREAD_EXACT_SIMT)
    assert torch.equal(i_tc, i_ex) and torch.equal(v_tc, v_ex) and torch.equal(o_tc, o_ex)
    assert bool((v_tc[..., :-1] >= v_tc[..., 1:]).all())
    assert int(i_tc.sort(-1)[0].diff(dim=-1).eq(0).sum()) == 0
    assert int(i_tc.min()) >= 0 and int(i_tc.max()) < slots
    bv.fill_(1.0)
    ones, _, _ = _read(bk, bv, slots, qk, k, ops.MEMREAD_TCGEN05)
    assert float((ones - 1).abs().max()) <= 1e-6
    # spot-check 64 (object, query) pairs against a float64 top-k of the full affinity row
    sel = torch.randint(0, K * hw, (64,), generator=torch.Generator().manual_seed(7))
    for s in sel.tolist():
        o, q = divmod(s, hw)
        aff = (bk[o].double() @ qk[q].double()) / (128 ** 0.5)
        ref = torch.topk(aff, k).indices.sort()[0]
        assert torch.equal(i_tc[o, q].long().sort()[0], ref)
    _lib.poll_kernel_error()
