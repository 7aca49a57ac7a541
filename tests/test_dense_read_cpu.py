"""CPU: the dense memory read of PropagationNetwork(top_k=None) without a GPU — its C ABI (declared, bound,
exported, the workspace query, argument checks that fail before any device call), the host runtime
(InferenceCore, LockstepSession) over a float64 stand-in of mivos_memory_read_dense registered here on top of
tests/abi_emulator.py, and the oracle's dense read against outputs of the unmodified reference
(tests/golden/dense.npz, oracle/gen_golden_dense.py)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import abi_emulator

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("mivos_memory_read_dense_workspace", "mivos_memory_read_dense")


def test_dense_symbols_declared_bound_and_exported():
    from mivos_b200 import _lib
    header = open(os.path.join(ROOT, "include", "mivos_b200.h")).read()
    lib = _lib.load()
    for name in NAMES:
        assert name + "(" in header and name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
    assert lib.mivos_abi_version() == 4


def test_dense_workspace_query_runs_without_a_gpu():
    from mivos_b200 import _lib
    lib = _lib.load()
    ws = lib.mivos_memory_read_dense_workspace
    one = ws(1, 21 * 1620, 1620)
    assert one > 0 and one % 256 == 0
    assert ws(4, 21 * 1620, 1620) >= 4 * (one - 256)  # per-object partials
    assert ws(5, 100 * 3600, 3600) < 2 ** 30  # cfg-5: well under 1 GB
    # the partition depends on hw alone: the workspace grows with the capacity, never with a live count
    assert ws(1, 2 * 21 * 1620, 1620) > one
    for bad in ((0, 100, 10), (257, 100, 10), (1, 0, 10), (1, 100, 0), (1, 1 << 31, 10)):
        assert ws(*bad) == -1, bad


def _call(lib, **kw):
    a = dict(bank_k=256, bank_v=256, slots_cap=100, k=1, slots=50, qk=256, hw=10, q_div=0, out=256, cstride=512,
             coff=0, hh=0, hw_=0, ws=256, ws_bytes=1 << 40, dyn=None, f16=0)
    a.update(kw)
    p = lambda v: C.c_void_p(v)  # noqa: E731  (never dereferenced: the checks come first)
    return lib.mivos_memory_read_dense(p(a["bank_k"]), p(a["bank_v"]), a["slots_cap"], a["k"], a["slots"], p(a["qk"]),
                                       a["hw"], a["q_div"], p(a["out"]), a["cstride"], a["coff"], a["hh"], a["hw_"],
                                       p(a["ws"]), a["ws_bytes"], p(a["dyn"]), a["f16"], p(0))


BAD_OPERANDS = [dict(bank_k=0), dict(slots=0), dict(slots=101), dict(k=0), dict(k=257), dict(hw=0),
                dict(q_div=-1), dict(cstride=510), dict(coff=4), dict(hh=3, hw_=4),
                dict(bank_v=260), dict(ws=272), dict(ws_bytes=1024)]


@pytest.mark.parametrize("bad", BAD_OPERANDS)
def test_dense_read_rejects_bad_arguments_before_any_device_call(bad):
    from mivos_b200 import _lib
    lib = _lib.load()
    assert _call(lib, **bad) == -1
    assert lib.mivos_last_error().decode().startswith("memory_read_dense")


def _call_topk(lib, **kw):
    a = dict(bank_k=256, bank_v=256, slots_cap=100, k=1, slots=50, qk=256, hw=10, q_div=0, top_k=20, out=256,
             cstride=512, coff=0, hh=0, hw_=0, ws=256, ws_bytes=1 << 40, algo=0, dyn=None, f16=0)
    a.update(kw)
    p = lambda v: C.c_void_p(v)  # noqa: E731  (never dereferenced: the checks come first)
    return lib.mivos_memory_read(p(a["bank_k"]), p(a["bank_v"]), a["slots_cap"], a["k"], a["slots"], p(a["qk"]), a["hw"],
                                 a["q_div"], a["top_k"], p(a["out"]), a["cstride"], a["coff"], a["hh"], a["hw_"], p(None),
                                 p(None), p(a["ws"]), a["ws_bytes"], a["algo"], p(a["dyn"]), a["f16"], p(0))


@pytest.mark.parametrize("bad", BAD_OPERANDS + [dict(cstride=1024, coff=-4), dict(qk=260), dict(top_k=0), dict(top_k=65),
                                                dict(algo=7)])
def test_topk_read_rejects_bad_arguments_before_any_device_call(bad):
    """The top-k read checks its operands by the rules of the dense read: a window that starts before the row
    (out_coff < 0) and a query pointer its kernels could not load as float4 are argument errors, not launches."""
    from mivos_b200 import _lib
    lib = _lib.load()
    assert _call_topk(lib, **bad) == -1
    assert lib.mivos_last_error().decode().startswith("memory_read:")


def test_dense_network_surface():
    import mivos_b200
    net = mivos_b200.PropagationNetwork(top_k=None)
    assert net.top_k is None and net.memory.top_k is None and net.attn_memory.top_k is None
    assert net.min_live_slots == 1 and mivos_b200.PropagationNetwork(top_k=20).min_live_slots == 20


# ------------------------------------------------------------------ host runtime over a float64 stand-in
def memory_read_dense_workspace_bytes(k, slots_cap, hw):
    return 16


def memory_read_dense(bank_k, bank_v, slots, qk, out, *, out_coff=0, halo_hw=None, workspace=None, dyn_slots=None,
                      q_div=0):
    """Header contract of mivos_memory_read_dense: per object, softmax over the live slots of keys . q / sqrt(128),
    weighted values (float64 inside).  Object o reads query set o // q_div of qk [sets,hw,128]."""
    k = bank_k.shape[0]
    if dyn_slots is not None:
        slots = int(dyn_slots[0])
    qsets = (qk if qk.dim() == 3 else qk[None]).float() / np.float32(128 ** 0.5)
    res = []
    for o in range(k):
        q = qsets[o // q_div if q_div > 0 else 0].double()
        w = torch.softmax(bank_k[o, :slots].double() @ q.t(), dim=0)  # [slots, hw]
        res.append((w.t() @ bank_v[o, :slots].double()).float())
    r = torch.stack(res)
    if halo_hw is not None:
        h, w_ = halo_hw
        out[:k, 1:-1, 1:-1, out_coff:out_coff + 512] = r.reshape(k, h, w_, 512).to(out.dtype)
    else:
        out[:, :, out_coff:out_coff + 512] = r.to(out.dtype)
    return out


@pytest.fixture()
def rt(monkeypatch, prop_sd, fuse_sd):
    mv = abi_emulator.install_host_runtime(monkeypatch)
    from mivos_b200 import ops
    monkeypatch.setattr(ops, "memory_read_dense_workspace_bytes", memory_read_dense_workspace_bytes)
    monkeypatch.setattr(ops, "memory_read_dense", memory_read_dense)
    net = mv.PropagationNetwork(top_k=None, act_dtype=torch.float32)
    net.load_state_dict(prop_sd, strict=True)
    fuse = mv.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    return mv, net, fuse


def _clip_lowres():
    from oracle import weights as Wt
    images, mask = Wt.synthetic_clip(6, 64, 88, 2, seed=21)
    _, mask2 = Wt.synthetic_clip(6, 64, 88, 2, seed=22)
    return images, mask, torch.roll(mask2, shifts=(5, 9), dims=(2, 3))


def _trace(g, j):
    return [tuple(int(x) for x in r) for r in g[f"clip_trace{j}"]]


def test_inference_core_host_runtime_matches_dense_golden(rt, golden):
    mv, net, fuse = rt
    g = golden("dense.npz")
    images, mask, mask2 = _clip_lowres()
    core = mv.InferenceCore(net, fuse, images, 2, mem_profile=0, mem_freq=2, device="cpu")
    m1 = core.interact(mask, 0)
    assert core.bank_trace == _trace(g, 1)
    d = (core.prob - torch.from_numpy(g["clip_prob1"])).abs()
    assert float(d.max()) <= 3e-2 and float(d.mean()) <= 1e-3
    assert float((m1 != g["clip_masks1"]).mean()) <= 0.01
    core.bank_trace = []
    m2 = core.interact(mask2, 5)  # fused second interaction
    assert core.bank_trace == _trace(g, 2)
    d = (core.prob - torch.from_numpy(g["clip_prob2"])).abs()
    assert float(d.max()) <= 3e-2 and float(d.mean()) <= 1e-3
    assert float((m2 != g["clip_masks2"]).mean()) <= 0.05


def test_lockstep_session_host_runtime_with_dense_read(rt):
    from oracle import weights as Wt
    mv, net, _ = rt
    C_, K, T = 3, 2, 7
    clips = [Wt.synthetic_clip(T, 64, 96, K, seed=40 + i) for i in range(C_)]
    solo = []
    for img, m in clips:
        core = mv.InferenceCore(net, None, img, K, mem_freq=2, device="cpu")
        core.interact(m, 2)
        solo.append(core)
    cores = [mv.InferenceCore(net, None, img, K, mem_freq=2, device="cpu") for img, _ in clips]
    out = mv.LockstepSession(cores).interact([m for _, m in clips], 2)
    for i in range(C_):
        assert cores[i].bank_trace == solo[i].bank_trace
        assert float((cores[i].prob - solo[i].prob).abs().max()) <= 1e-4
        assert (out[i] == solo[i].np_masks).mean() >= 0.9999


def test_dense_read_guard_accepts_one_live_slot(rt):
    """The live-slot guard asks the network: a dense read needs one live slot, not top_k of them."""
    mv, net, _ = rt
    assert net.min_live_slots == 1
    from oracle import weights as Wt
    images, mask = Wt.synthetic_clip(3, 16, 16, 1, seed=3)  # one bank slot per frame
    core = mv.InferenceCore(net, None, images, 1, mem_freq=1, device="cpu")
    core.interact(mask, 0)
    assert core.bank_trace[0] == (1, 1)


# ------------------------------------------------------------------ the oracle against the reference's outputs
def test_oracle_dense_read_matches_reference(golden):
    from oracle import stm_oracle as O
    from oracle.gen_golden_dense import MEMREAD_CASES, memread_inputs
    g = golden("dense.npz")
    for name, (K, T, seed) in MEMREAD_CASES.items():
        mk, mv, qk = memread_inputs(K, T, seed)
        assert torch.equal(O.memory_read(mk, mv, qk, None), torch.from_numpy(g[f"memread_{name}_out"])), name


def test_oracle_inference_core_dense_matches_reference(prop_sd, fuse_sd, golden):
    from oracle import stm_oracle as O
    g = golden("dense.npz")
    images, mask, _ = _clip_lowres()
    oc = O.OracleInferenceCore(prop_sd, fuse_sd, images, 2, mem_freq=2, top_k=None)
    m = oc.interact(mask, 0)
    assert torch.equal(oc.prob, torch.from_numpy(g["clip_prob1"])) and (m == g["clip_masks1"]).all()
    assert oc.bank_trace == _trace(g, 1)
