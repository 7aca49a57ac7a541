"""CPU: the wide top-k memory read of PropagationNetwork(top_k=k), 64 < k <= 1024, without a GPU — its C ABI
(declared, bound, exported, the workspace query, argument checks that fail before any device call), the routing of
PropagationEngine._memory_read, and the host runtime (InferenceCore, LockstepSession) over a float64 stand-in of
mivos_memory_read_wide registered here on top of tests/abi_emulator.py, checked against the float64 oracle."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import abi_emulator

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("mivos_memory_read_wide_workspace", "mivos_memory_read_wide")


def test_wide_symbols_declared_bound_and_exported():
    from mivos_b200 import _lib
    header = open(os.path.join(ROOT, "include", "mivos_b200.h")).read()
    lib = _lib.load()
    for name in NAMES:
        assert name + "(" in header and name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
    assert len(_lib.SIGNATURES["mivos_memory_read_wide"][1]) == 21
    assert len(_lib.SIGNATURES["mivos_memory_read_wide_workspace"][1]) == 4
    assert lib.mivos_abi_version() == 4


def test_wide_workspace_query_runs_without_a_gpu():
    from mivos_b200 import _lib
    ws = _lib.load().mivos_memory_read_wide_workspace
    one = ws(1, 20 * 1620, 1620, 128)
    assert one > 0
    # it depends on (objects, hw): not on the capacity, nor on k
    assert ws(1, 40 * 1620, 1620, 128) == one == ws(1, 20 * 1620, 1620, 1024) == ws(1, 20 * 1620, 1620, 1)
    assert ws(5, 100 * 3600, 3600, 1024) < 2 ** 30
    for bad in ((0, 100, 10, 100), (257, 100, 10, 100), (1, 0, 10, 100), (1, 100, 0, 100), (1, 1 << 31, 10, 100),
                (1, 2000, 10, 0), (1, 2000, 10, 1025)):
        assert ws(*bad) == -1, bad


def _call(lib, **kw):
    a = dict(bank_k=256, bank_v=256, slots_cap=2000, k=1, slots=1500, qk=256, hw=10, q_div=0, top_k=100, out=256,
             cstride=512, coff=0, hh=0, hw_=0, ws=256, ws_bytes=1 << 40, dyn=None, f16=0)
    a.update(kw)
    p = lambda v: C.c_void_p(v)  # noqa: E731  (never dereferenced: the checks come first)
    return lib.mivos_memory_read_wide(p(a["bank_k"]), p(a["bank_v"]), a["slots_cap"], a["k"], a["slots"], p(a["qk"]),
                                      a["hw"], a["q_div"], a["top_k"], p(a["out"]), a["cstride"], a["coff"], a["hh"],
                                      a["hw_"], p(None), p(None), p(a["ws"]), a["ws_bytes"], p(a["dyn"]), a["f16"], p(0))


# the dense read's bad-operand list (tests/test_dense_read_cpu.py), plus the top-k read's extra cases and the wide
# read's own: k = 0, k = 1025, fewer live slots than k
BAD_OPERANDS = [dict(bank_k=0), dict(slots=0), dict(slots=2001), dict(k=0), dict(k=257), dict(hw=0),
                dict(q_div=-1), dict(cstride=510), dict(coff=4), dict(hh=3, hw_=4),
                dict(bank_v=260), dict(ws=272), dict(ws_bytes=1024), dict(cstride=1024, coff=-4), dict(qk=260),
                dict(top_k=0), dict(top_k=1025), dict(slots=99), dict(slots=1023, slots_cap=1025, top_k=1024)]


@pytest.mark.parametrize("bad", BAD_OPERANDS)
def test_wide_read_rejects_bad_arguments_before_any_device_call(bad):
    from mivos_b200 import _lib
    lib = _lib.load()
    assert _call(lib, **bad) == -1
    assert lib.mivos_last_error().decode().startswith("memory_read_wide")


def test_topk_read_still_rejects_65():
    from mivos_b200 import _lib
    lib = _lib.load()
    assert lib.mivos_memory_read_workspace(1, 2000, 10, 65) == -1
    p = C.c_void_p
    rc = lib.mivos_memory_read(p(256), p(256), 2000, 1, 1500, p(256), 10, 0, 65, p(256), 512, 0, 0, 0, p(None), p(None),
                               p(256), 1 << 40, 0, p(None), 0, p(0))
    assert rc == -1 and lib.mivos_last_error().decode().startswith("memory_read:")


# ------------------------------------------------------------------ host runtime over a float64 stand-in
CALLS = []


def _read64(bank_k, bank_v, slots, qk, top_k, out, out_coff, halo_hw, dyn_slots, q_div):
    """Header contract of the top-k reads: per object, top_k of keys . q / sqrt(128) over the live slots (score desc,
    slot asc), softmax over them, weighted values (float64 inside).  Object o reads query set o // q_div."""
    k = bank_k.shape[0]
    if dyn_slots is not None:
        slots = int(dyn_slots[0])
    qsets = (qk if qk.dim() == 3 else qk[None]).float() / np.float32(128 ** 0.5)
    res = []
    for o in range(k):
        q = qsets[o // q_div if q_div > 0 else 0].double()
        aff = bank_k[o, :slots].double() @ q.t()  # [slots, hw]
        vals, ind = torch.topk(aff, top_k, dim=0)
        w = torch.softmax(vals, dim=0)  # [k, hw]
        res.append(torch.einsum("jq,jqc->qc", w, bank_v[o].double()[ind]).float())
    r = torch.stack(res)
    if halo_hw is not None:
        h, w_ = halo_hw
        out[:k, 1:-1, 1:-1, out_coff:out_coff + 512] = r.reshape(k, h, w_, 512).to(out.dtype)
    else:
        out[:, :, out_coff:out_coff + 512] = r.to(out.dtype)
    return out


def memory_read_wide_workspace_bytes(k, slots_cap, hw, top_k):
    if not 1 <= top_k <= 1024:
        from mivos_b200 import _lib
        raise _lib.MivosError("memory_read_wide_workspace: bad arguments")
    return 16


def memory_read_wide(bank_k, bank_v, slots, qk, top_k, out, *, out_coff=0, halo_hw=None, workspace=None,
                     want_topk=False, dyn_slots=None, q_div=0):
    CALLS.append(("wide", top_k))
    return _read64(bank_k, bank_v, slots, qk, top_k, out, out_coff, halo_hw, dyn_slots, q_div)


@pytest.fixture()
def rt(monkeypatch, prop_sd, fuse_sd):
    mv = abi_emulator.install_host_runtime(monkeypatch)
    from mivos_b200 import ops
    monkeypatch.setattr(ops, "memory_read_wide_workspace_bytes", memory_read_wide_workspace_bytes)
    monkeypatch.setattr(ops, "memory_read_wide", memory_read_wide)
    # the stand-ins of the other two reads only record that they were chosen
    monkeypatch.setattr(ops, "memory_read", lambda *a, **kw: CALLS.append(("topk", a[4])))
    monkeypatch.setattr(ops, "memory_read_workspace_bytes", lambda *a: 16)
    monkeypatch.setattr(ops, "memory_read_dense", lambda *a, **kw: CALLS.append(("dense", None)))
    monkeypatch.setattr(ops, "memory_read_dense_workspace_bytes", lambda *a: 16)
    CALLS.clear()

    def make(top_k):
        net = mv.PropagationNetwork(top_k=top_k, act_dtype=torch.float32)
        net.load_state_dict(prop_sd, strict=True)
        return net
    fuse = mv.FusionNet()
    fuse.load_state_dict(fuse_sd, strict=True)
    return mv, make, fuse


def _clip(T=6, h=128, w=176, K=2, seed=21):
    from oracle import weights as Wt
    return Wt.synthetic_clip(T, h, w, K, seed=seed)


@pytest.mark.parametrize("top_k,which", [(100, "wide"), (50, "topk"), (None, "dense")])
def test_engine_routes_each_top_k_to_one_read(rt, top_k, which):
    mv, make, _ = rt
    images, mask = _clip(T=4, h=192, w=256)  # 192 slots per frame
    net = make(top_k)
    assert net.min_live_slots == (1 if top_k is None else top_k)
    mv.InferenceCore(net, None, images, 2, mem_freq=1, device="cpu").interact(mask, 0)
    assert CALLS and {c[0] for c in CALLS} == {which}


def test_top_k_past_the_cap_is_refused(rt):
    """1025 live slots pass the live-slot guard; the engine refuses the top_k itself."""
    from mivos_b200 import _lib
    mv, make, _ = rt
    images, mask = _clip(T=2, h=512, w=528, K=1)  # 32 x 33 = 1056 slots per frame
    core = mv.InferenceCore(make(1025), None, images, 1, mem_freq=1, device="cpu")
    with pytest.raises(_lib.MivosError, match="largest served top_k"):
        core.interact(mask, 0)
    assert not CALLS


def _trace(g, j):
    return [tuple(int(x) for x in r) for r in g[f"clip_trace{j}"]]


def test_inference_core_with_the_wide_read_matches_reference_golden(rt, golden):
    from oracle import gen_golden_wide as GW
    mv, make, fuse = rt
    g = golden("wide.npz")
    images, mask, mask2 = GW.clip_inputs()
    core = mv.InferenceCore(make(GW.CLIP_TOP_K), fuse, images, 2, mem_profile=0, mem_freq=2, device="cpu")
    m1 = core.interact(mask, 0)
    assert core.bank_trace == _trace(g, 1)
    d = (core.prob - torch.from_numpy(g["clip_prob1"])).abs()
    assert float(d.max()) <= 3e-2 and float(d.mean()) <= 1e-3
    assert float((m1 != g["clip_masks1"]).mean()) <= 0.01
    core.bank_trace = []
    m2 = core.interact(mask2, images.shape[1] - 1)  # fused second interaction
    assert core.bank_trace == _trace(g, 2)
    d = (core.prob - torch.from_numpy(g["clip_prob2"])).abs()
    assert float(d.max()) <= 3e-2 and float(d.mean()) <= 1e-3
    assert float((m2 != g["clip_masks2"]).mean()) <= 0.05
    assert {c[0] for c in CALLS} == {"wide"}


def test_lockstep_session_with_the_wide_read(rt):
    mv, make, _ = rt
    net = make(100)
    C_, K, T = 3, 2, 6
    clips = [_clip(T, 192, 256, K, seed=40 + i) for i in range(C_)]
    solo = []
    for img, m in clips:
        core = mv.InferenceCore(net, None, img, K, mem_freq=1, device="cpu")
        core.interact(m, 1)
        solo.append(core)
    cores = [mv.InferenceCore(net, None, img, K, mem_freq=1, device="cpu") for img, _ in clips]
    out = mv.LockstepSession(cores).interact([m for _, m in clips], 1)
    for i in range(C_):
        assert cores[i].bank_trace == solo[i].bank_trace
        assert float((cores[i].prob - solo[i].prob).abs().max()) <= 1e-4
        assert (out[i] == solo[i].np_masks).mean() >= 0.9999


# ------------------------------------------------------------------ the oracle against the reference's outputs
def test_oracle_wide_read_matches_reference(golden):
    from oracle import gen_golden_wide as GW
    from oracle import stm_oracle as O
    g = golden("wide.npz")
    for k in GW.MEMREAD_K:
        for K in GW.MEMREAD_OBJECTS:
            mk, mv, qk = GW.memread_inputs(K, k, GW.memread_seed(K, k))
            o = torch.cat([O.memory_read(mk[i:i + 1], mv[i:i + 1], qk, k) for i in range(K)], 0)  # one object per read
            assert torch.equal(o, torch.from_numpy(g[f"memread_k{k}_K{K}_out"])), (k, K)


def test_oracle_segment_with_query_matches_reference(prop_sd, golden):
    from oracle import gen_golden_wide as GW
    from oracle import stm_oracle as O
    mk, mv, qv = GW.seg_inputs(golden("reference_live.npz"))
    assert torch.equal(O.segment_with_query(prop_sd, mk, mv, *qv, GW.SEG_TOP_K), torch.from_numpy(golden("wide.npz")["seg_out"]))
