"""CPU: the memory census checker (tests/memory_census.py) has teeth.

The emulated reads and bank writes of tests/abi_emulator*.py pass it, in every layout (scalar with q_div, per-set,
object groups) and into fp32 and fp16 HALO windows of a larger allocation, and so does a kernel that swaps two slots
whose float64 scores tie.  Each emulated kernel bug fails it: a group read with its neighbour's count, the last live
slot never selected, a softmax over k - 1 of the k selected slots, a swap outside TIE_EPS, one element written to map N
or to channel 512 of `cat`, a dense read without the O rescale, and bank writes to the wrong frame or rows."""
import math

import pytest
import torch

import abi_emulator as E
import abi_emulator_groups as EG
import abi_emulator_sets as ES
import memory_census as MC
from test_gpu_memread_dense import TILE, _teeth_data

H16, F32 = torch.float16, torch.float32
h, w = 5, 7
HW = h * w
CAP = 4 * HW


def _bank(maps, seed, counts=None):
    """N(0, 1) keys with a common component (as the key projection gives), values; slots past each map's live count
    hold keys that would outrank every live slot."""
    g = torch.Generator().manual_seed(seed)
    bk = torch.randn((maps, CAP, 128), generator=g) * 0.5 + torch.randn((1, 1, 128), generator=g)
    bv = torch.randn((maps, CAP, 512), generator=g)
    if counts is not None:
        for o, n in enumerate(counts):
            bk[o, n:] = 8.0 * bk[o, :1].abs()
    return bk, bv


def _qk(sets, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((sets, HW, 128), generator=g) + torch.randn((1, 1, 128), generator=g)


def _cat(maps, dtype, extra=2):
    """A `cat` map of `maps` maps as the leading view of an allocation of maps + extra maps, filled with a sentinel."""
    parent = torch.full((maps + extra, h + 2, w + 2, 1024), -3.5, dtype=dtype)
    return parent, parent[:maps]


def _first(sizes):
    f = [0]
    for k in sizes:
        f.append(f[-1] + k)
    return torch.tensor(f, dtype=torch.int32)


SIZES = [2, 1, 3]          # object groups: a one-object group in the middle
COUNTS = [3 * HW - 5, HW + 3, 2 * HW]


def _groups_args(dtype=F32, k=5, seed=1):
    maps = sum(SIZES)
    live = [c for n, c in zip(SIZES, COUNTS) for _ in range(n)]
    bk, bv = _bank(maps, seed, live)
    parent, cat = _cat(maps, dtype)
    return dict(bank_k=bk, bank_v=bv, slots=CAP, qk=_qk(len(SIZES), seed + 1), top_k=k, out=cat,
                counts=torch.tensor(COUNTS, dtype=torch.int32), first=_first(SIZES), halo_hw=(h, w)), parent


# ------------------------------------------------------------------ the emulators pass
@pytest.mark.parametrize("dtype", [F32, H16], ids=["f32", "f16"])
def test_emulated_reads_pass(dtype):
    A, _ = _groups_args(dtype)
    rec = MC.checked_read("memory_read_groups", EG.memory_read_groups, A)
    assert rec["ratio"] <= 1.0 and rec["layout"] == "groups" and rec["parts"] == 6 and rec["live"][2] == HW + 3
    bk, bv = _bank(4, 3, [2 * HW + 1] * 4)
    _, cat = _cat(4, dtype)
    A = dict(bank_k=bk, bank_v=bv, slots=CAP, qk=_qk(2, 4), top_k=20, out=cat, counts=torch.tensor(
        [2 * HW + 1, 2 * HW + 1], dtype=torch.int32), halo_hw=(h, w))
    assert MC.checked_read("memory_read_sets", ES.memory_read_sets, A)["ratio"] <= 1.0
    A = dict(bank_k=bk, bank_v=bv, slots=CAP, qk=_qk(2, 4), top_k=20, out=cat, halo_hw=(h, w), q_div=2,
             dyn_slots=torch.tensor([2 * HW + 1], dtype=torch.int32))
    rec = MC.checked_read("memory_read", E.memory_read, A, max_scores=0)  # the sampled path
    assert rec["ratio"] <= 1.0 and rec["sampled"] and rec["q_div"] == 2 and rec["device_count"]


def test_sample_queries_cover_tile_edges():
    hw = 1000
    got = set(MC.sample_queries(hw, seed=2).tolist())
    assert set(range(64)) | set(range(960, 1000)) <= got and max(got) < hw
    for m0 in range(0, hw, 64):
        assert {m0, m0 + 31, m0 + 32, m0 + 63} & set(range(hw)) <= got
    assert len(got) >= min(hw, MC.SAMPLE_RANDOM) * 0.9


# ------------------------------------------------------------------ mutated top-k kernels
def _topk_kernel(mutate):
    """memory_read_groups over the header's contract in float32 with a bug injected by mutate(stage, value)."""
    def kernel(bank_k, bank_v, slots, qk, top_k, out, counts, first, *, out_coff=0, halo_hw=None, workspace=None,
               algo=0, want_topk=False):
        f = [int(v) for v in first]
        cnt = mutate("counts", [int(v) for v in counts])
        sel = []
        for g in range(len(f) - 1):
            for o in range(f[g], f[g + 1]):
                n = mutate("live", cnt[g])
                aff = bank_k[o, :n] @ (qk[g] / math.sqrt(128)).t()          # [n, hw]
                vals, idx = torch.topk(aff, top_k + 1, dim=0)
                idx = mutate("idx", idx[:top_k].clone(), idx[top_k])
                used = mutate("used", idx)
                wgt = torch.softmax(aff.gather(0, used), dim=0)
                r = torch.einsum("kq,kqc->qc", wgt, bank_v[o][used])
                out[o, 1:-1, 1:-1, out_coff:out_coff + 512] = r.reshape(h, w, 512).to(out.dtype)
                sel.append(idx.t().int())
        mutate("out", out)
        return (out, torch.stack(sel), None) if want_topk else out
    return kernel


def _none(stage, v, *rest):
    return v


def _neighbour_count(stage, v, *rest):
    return v[-1:] + v[:-1] if stage == "counts" else v


def _last_slot_dropped(stage, v, *rest):
    return v - 1 if stage == "live" else v


def _softmax_k_minus_1(stage, v, *rest):
    return v[:-1] if stage == "used" else v


def _swap_kth(stage, v, *rest):
    if stage == "idx":
        v[-1] = rest[0]   # the (k+1)-th slot in place of the k-th
    return v


def _spill_to_map_n(parent, maps):
    def mutate(stage, v, *rest):
        if stage == "out":
            parent[maps, 3, 4, 100] = 0.25
        return v
    return mutate


def _spill_to_channel_512(stage, v, *rest):
    if stage == "out":
        v[1, 2, 2, 512] = 0.25
    return v


def test_unmutated_kernel_passes():
    A, _ = _groups_args()
    assert MC.checked_read("memory_read_groups", _topk_kernel(_none), A)["ratio"] <= 1.0


def test_last_live_slot_in_the_top_k():
    """Data for the dropped-last-slot mutation: each group's last live slot outranks every other live slot."""
    A, _ = _groups_args()
    bk, qk, f = A["bank_k"], A["qk"], [int(v) for v in A["first"]]
    for g in range(len(SIZES)):
        bk[f[g]:f[g + 1], COUNTS[g] - 1] = 3.0 * qk[g].mean(0)
    assert MC.checked_read("memory_read_groups", _topk_kernel(_none), A)["ratio"] <= 1.0
    A2, _ = _groups_args()
    A2["bank_k"] = bk
    with pytest.raises(AssertionError, match="another top-5 set"):
        MC.checked_read("memory_read_groups", _topk_kernel(_last_slot_dropped), A2)


@pytest.mark.parametrize("mutation,match", [
    (_neighbour_count, "another top-5 set|outside \\[0"),
    (_softmax_k_minus_1, "exceeds the bound"),
    (_swap_kth, "another top-5 set"),
    (_spill_to_channel_512, "outside its window"),
], ids=["neighbours_count", "softmax_over_k_minus_1", "swap_outside_tie_eps", "channel_512_of_cat"])
def test_mutated_read_fails(mutation, match):
    A, _ = _groups_args()
    with pytest.raises(AssertionError, match=match):
        MC.checked_read("memory_read_groups", _topk_kernel(mutation), A)


def test_write_into_map_n_fails():
    A, parent = _groups_args()
    with pytest.raises(AssertionError, match="outside its window"):
        MC.checked_read("memory_read_groups", _topk_kernel(_spill_to_map_n(parent, sum(SIZES))), A)


def test_swap_within_tie_eps_passes():
    """Every key duplicated: the k-th and (k+1)-th slots of each query tie (k odd), and a kernel that swaps them
    is right — its read-out is checked over its own set."""
    A, _ = _groups_args(k=5)
    bk = A["bank_k"]
    bk[:, 1::2] = bk[:, 0::2]
    rec = MC.checked_read("memory_read_groups", _topk_kernel(_swap_kth), A)
    assert rec["ratio"] <= 1.0 and rec["swaps"] > 0 and rec["ties"] > 0


# ------------------------------------------------------------------ dense reads
def _dense_kernel(rescale):
    """memory_read_dense by an online softmax over 32-slot tiles (float64, output fp32); rescale=False drops the
    rescale of O when the running maximum grows (l is rescaled)."""
    def kernel(bank_k, bank_v, slots, qk, out, *, out_coff=0, halo_hw=None, workspace=None, dyn_slots=None,
               q_div=0):
        n = int(dyn_slots[0]) if dyn_slots is not None else slots
        q = MC.scaled_q(qk)
        for o in range(bank_k.shape[0]):
            s = bank_k[o, :n].double() @ q.t()
            v = bank_v[o, :n].double()
            m = torch.full((q.shape[0],), -math.inf, dtype=torch.float64)
            l, acc = torch.zeros_like(m), torch.zeros((q.shape[0], 512), dtype=torch.float64)
            for t0 in range(0, n, TILE):
                st = s[t0:t0 + TILE]
                m_new = torch.maximum(m, st.amax(0))
                p = torch.exp(st - m_new)
                l = l * torch.exp(m - m_new) + p.sum(0)
                acc = (acc * torch.exp(m - m_new)[:, None] if rescale else acc) + p.t() @ v[t0:t0 + TILE]
                m = m_new
            out[o, :, out_coff:out_coff + 512] = (acc / l[:, None]).to(out.dtype)
        return out
    return kernel


def test_dense_read_without_the_o_rescale_fails():
    bk, bv, qk = _teeth_data()
    n = bk.shape[0]
    A = dict(bank_k=bk[None].contiguous(), bank_v=bv[None].contiguous(), slots=n, qk=qk,
             out=torch.full((1, qk.shape[0], 1024), 9.0))
    assert MC.checked_read("memory_read_dense", _dense_kernel(True), dict(A, out=A["out"].clone()))["ratio"] <= 1.0
    with pytest.raises(AssertionError, match="dense read's bound"):
        MC.checked_read("memory_read_dense", _dense_kernel(False), A)


# ------------------------------------------------------------------ bank writes
def _write_args(form, seed=5):
    g = torch.Generator().manual_seed(seed)
    maps = sum(SIZES) if form == "groups" else 6
    halo = torch.randn((maps, h + 2, w + 2, 640), generator=g)
    parent_k = torch.full((maps + 2, CAP, 128), 1.5)
    parent_v = torch.full((maps + 2, CAP, 512), -1.5)
    bk, bv = parent_k[1:1 + maps], parent_v[1:1 + maps]  # a slice of a larger bank that does not start at map 0
    A = dict(halo=halo, h=h, w=w, coff_k=0, coff_v=128, bank_k=bk, bank_v=bv)
    if form == "scalar":
        A.update(k=maps, t=3, dyn_t=torch.tensor([2], dtype=torch.int32))
    elif form == "sets":
        A.update(k=maps, sets=3, t_max=3, dyn_t=torch.tensor([1, 5, 3], dtype=torch.int32))  # frame 5: no write
    else:
        A.update(n=maps, t_max=3, dyn_t=torch.tensor([0, 2, 3], dtype=torch.int32), first=_first(SIZES))
    return A


EMULATED_WRITES = {"scalar": ("bank_write", E.bank_write), "sets": ("bank_write_sets", ES.bank_write_sets),
                   "groups": ("bank_write_groups", EG.bank_write_groups)}


@pytest.mark.parametrize("layout", list(EMULATED_WRITES))
def test_emulated_writes_pass(layout):
    form, fn = EMULATED_WRITES[layout]
    rec = MC.checked_write(form, fn, _write_args(layout))
    assert rec["form"] == form and rec["frames"][0] in (0, 1, 2)


def test_write_outside_t_max_writes_nothing():
    A = _write_args("sets")
    before = A["bank_k"].clone()
    MC.checked_write("bank_write_sets", ES.bank_write_sets, A)
    assert torch.equal(A["bank_k"][2:4], before[2:4])  # set 1's frame 5 lies past t_max = 3


def _groups_next_frame(halo, n, h, w, coff_k, coff_v, bank_k, bank_v, t_max, dyn_t, first):
    EG.bank_write_groups(halo, n, h, w, coff_k, coff_v, bank_k, bank_v, t_max, dyn_t + 1, first)


def _groups_into_next_rows(halo, n, h, w, coff_k, coff_v, bank_k, bank_v, t_max, dyn_t, first):
    """Group 0 writes its maps into group 1's rows (its own frame), the other groups as they should."""
    f = [int(v) for v in first]
    for g in range(len(f) - 1):
        a, b = f[g], f[g + 1]
        d = f[1] if g == 0 else a
        E.bank_write(halo[a:b], b - a, h, w, coff_k, coff_v, bank_k[d:d + b - a], bank_v[d:d + b - a], int(dyn_t[g]))


@pytest.mark.parametrize("kernel", [_groups_next_frame, _groups_into_next_rows], ids=["frame_plus_1", "next_groups_rows"])
def test_mutated_write_fails(kernel):
    with pytest.raises(AssertionError, match="differs from the expected write"):
        MC.checked_write("bank_write_groups", kernel, _write_args("groups"))


def test_census_records_emulated_launches(monkeypatch):
    """MemoryCensus.record swaps the twelve ops attributes, checks each new launch once and restores them."""
    from mivos_b200 import ops
    E.install(monkeypatch, ops)
    EG.install(monkeypatch, ops)
    census = MC.MemoryCensus()
    A, _ = _groups_args()
    W = _write_args("groups")
    with census.record("emulated"):
        for _ in range(2):
            ops.memory_read_groups(**A)
            ops.bank_write_groups(**W)
    assert census.seen["emulated"] == 4 and census.checked["emulated"] == 2
    assert ops.memory_read_groups is EG.memory_read_groups and ops.bank_write_groups is EG.bank_write_groups
    assert len(census.records) == 1 and len(census.writes) == 1
    print("\n" + census.table() + "\n" + census.summary())
