"""TEST INFRASTRUCTURE: the memory census — every memory read and bank write of a real session, checked on its own
operands (keys from the key projection, banks written at per-clip frames, HALO `cat` windows in fp16 and fp32, and
the q_div / per-set / object-group layouts) against float64 restatements of include/mivos_b200.h.

Each read launch's objects get their query set and live slot count from the launch's own arguments: the scalar
`slots` or dyn_slots[0] with q_div, o // (K / sets) with counts[s], or the group of o in `first` with counts[g]
(device tables are read after the synchronisation; counts are clamped to the capacity).  Checks (DESIGN.md section 6):
  top-k and wide reads
    1. the launch re-run with want_topk into a scratch output and a fresh workspace gives the production bits; the
       top-k forms (memory_read, _sets, _groups) re-run with MEMREAD_EXACT_SIMT give them too;
    2. against float64 scores (q divided by sqrt(128) in fp32, as the reference): the indices are unique and below
       the object's live count; the index set equals the float64 top-k wherever the k-th/(k+1)-th gap exceeds
       TIE_EPS; everywhere the smallest float64 score of the chosen set is at least the k-th score - TIE_EPS;
    3. for every query, near-ties included, the read-out is the float64 softmax read-out over the kernel's own chosen
       set within RANGE_TERM of the launch's output range (+ ROUND_TERM |ref| into an fp16 `cat`);
  dense reads: the elementwise bound of tests/test_gpu_memread_dense.py (its `reference`), every query, + ROUND_TERM
    |ref| into an fp16 `cat`;
  every read: the window is finite, and every byte of the output's whole allocation outside interior rows x
    channels [out_coff, out_coff + 512) of the maps that take part keeps its value (maps no group holds and maps past
    a lock-step tick's prefix take part in nothing);
  every bank write: the rows of frame dyn_t[g] (or t) of group / set g's maps hold the interior key and value channels
    of the source map bit for bit, a frame outside [0, t_max] writes nothing, and no other byte of either bank's
    allocation changes.  Banks above BANK_SNAPSHOT_BYTES (a 1080p clip's bank) are not cloned: the write is counted,
    not checked.
Top-k and wide reads above SAMPLE_SCORES float64 scores check a deterministic sample of queries (`sample_queries`).
For the top-k forms the TF32 candidate path's statistics (mivos_memory_read_stats) are recorded, not asserted.

`MemoryCensus.record(scenario)` replaces the twelve ops attributes the engine calls through; launches are
deduplicated by (form, K, hw, capacity, top_k, output type, live counts, `first`, q_div).  Importable without a GPU:
tests/test_memory_census_cpu.py drives `checked_read` / `checked_write` with emulated kernels and their mutations."""
from __future__ import annotations

import contextlib
import ctypes as C
import inspect
import math
from collections import Counter
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import torch

from conv_census import changed_outside, like, storage_bytes

TIE_EPS = 1e-5              # float64 score gap below which fp32 summation order may decide the top-k set
RANGE_TERM = 2e-5           # of the launch's max|ref|: fp32 round-off of a k-term weighted sum
ROUND_TERM = 2.0 ** -11     # of |ref|: one rounding into an fp16 `cat`
SAMPLE_SCORES = 2 ** 28     # maps x live slots x queries above which a top-k / wide read checks sampled queries
SAMPLE_RANDOM = 4096
Q_TILE = 64
BANK_SNAPSHOT_BYTES = 512 << 20  # bank_k + bank_v allocations above which a bank write is counted, not checked
C_OUT = 512

READS = {
    "memory_read": ("topk", "scalar"), "memory_read_sets": ("topk", "sets"), "memory_read_groups": ("topk", "groups"),
    "memory_read_dense": ("dense", "scalar"), "memory_read_dense_sets": ("dense", "sets"),
    "memory_read_dense_groups": ("dense", "groups"),
    "memory_read_wide": ("wide", "scalar"), "memory_read_wide_sets": ("wide", "sets"),
    "memory_read_wide_groups": ("wide", "groups"),
}
WRITES = {"bank_write": "scalar", "bank_write_sets": "sets", "bank_write_groups": "groups"}


def _ints(t) -> list:
    return [int(v) for v in t.reshape(-1).cpu().tolist()]


def bind(fn, args, kw) -> dict:
    """The launch's arguments by name, defaults included."""
    b = inspect.signature(fn).bind(*args, **kw)
    b.apply_defaults()
    return dict(b.arguments)


def sample_queries(hw: int, seed: int = 0) -> torch.Tensor:
    """The first and last 64-query tiles, queries 0, 31, 32 and 63 of every tile, SAMPLE_RANDOM seeded queries."""
    tiles = -(-hw // Q_TILE)
    parts = [torch.arange(0, Q_TILE), torch.arange((tiles - 1) * Q_TILE, tiles * Q_TILE)]
    m0 = torch.arange(tiles) * Q_TILE
    parts += [m0 + d for d in (0, 31, 32, 63)]
    parts.append(torch.randint(0, hw, (SAMPLE_RANDOM,), generator=torch.Generator().manual_seed(seed)))
    r = torch.unique(torch.cat(parts))
    return r[r < hw]


def scaled_q(qk: torch.Tensor) -> torch.Tensor:
    """q / sqrt(128) in fp32, as the reference divides, then float64."""
    return (qk.float() / np.float32(math.sqrt(128))).double()


# ------------------------------------------------------------------ reads
@dataclass
class ReadLaunch:
    form: str
    kind: str                  # topk | wide | dense
    layout: str                # scalar | sets | groups
    fn: object                 # the launch function (the real operator, or an emulation on the CPU)
    args: dict
    maps: int
    hw: int
    cap: int
    top_k: Optional[int]
    qset: list                 # query set of each map (-1: the map takes part in nothing)
    live: list                 # live slots of each map
    counts: tuple              # the live counts of the launch: (n,) scalar, one per set / group
    first: Optional[tuple]
    q_div: int
    before: Optional[torch.Tensor] = None

    @property
    def out(self) -> torch.Tensor:
        return self.args["out"]

    @property
    def sig(self) -> tuple:
        return (self.form, self.maps, self.hw, self.cap, self.top_k, self.out.dtype, self.counts, self.first,
                self.q_div)

    @property
    def tag(self) -> str:
        return (f"{self.form} (K {self.maps}, hw {self.hw}, cap {self.cap}, k {self.top_k}, counts {self.counts}, "
                f"first {self.first}, q_div {self.q_div}, {'f16' if self.out.dtype == torch.float16 else 'f32'} out)")


def read_launch(form: str, fn, A: dict) -> ReadLaunch:
    """The launch's objects, query sets and live counts (device tables read here: synchronise first)."""
    kind, layout = READS[form]
    bk, qk = A["bank_k"], A["qk"]
    K, cap = bk.shape[0], bk.shape[1]
    hw = qk.shape[-2]
    top_k = A.get("top_k")
    first = None
    if layout == "scalar":
        n = _ints(A["dyn_slots"])[0] if A.get("dyn_slots") is not None else int(A["slots"])
        q_div = int(A.get("q_div") or 0)
        qset = [o // q_div if q_div else 0 for o in range(K)]
        counts = (n,)
        live = [min(max(n, 0), cap)] * K
    elif layout == "sets":
        sets = qk.shape[0]
        q_div = K // sets
        counts = tuple(_ints(A["counts"])[:sets])
        qset = [o // q_div for o in range(K)]
        live = [min(max(counts[s], 0), cap) for s in qset]
    else:
        q_div = 0
        first = tuple(_ints(A["first"]))
        counts = tuple(_ints(A["counts"])[:len(first) - 1])
        qset = [-1] * K
        for g in range(len(first) - 1):
            for o in range(max(first[g], 0), min(first[g + 1], K)):
                qset[o] = g
        live = [min(max(counts[g], 0), cap) if g >= 0 else 0 for g in qset]
    return ReadLaunch(form, kind, layout, fn, A, K, hw, cap, top_k, qset, live, counts, first, q_div)


def _runs(qset) -> list:
    """Maximal runs [a, b) of maps that take part."""
    out, a = [], None
    for o, s in enumerate(list(qset) + [-1]):
        if s >= 0 and a is None:
            a = o
        elif s < 0 and a is not None:
            out.append((a, o))
            a = None
    return out


def read_windows(L: ReadLaunch, t: torch.Tensor) -> list:
    """The written windows of an output laid out as L's: interior x [out_coff, out_coff + 512) of the maps that
    take part."""
    c0 = L.args.get("out_coff", 0)
    if L.args.get("halo_hw") is not None:
        return [t[a:b, 1:-1, 1:-1, c0:c0 + C_OUT] for a, b in _runs(L.qset)]
    return [t[a:b, :, c0:c0 + C_OUT] for a, b in _runs(L.qset)]


def map_rows(L: ReadLaunch, t: torch.Tensor, o: int) -> torch.Tensor:
    """Map o's read-out [hw, 512] in the output t."""
    c0 = L.args.get("out_coff", 0)
    if L.args.get("halo_hw") is not None:
        return t[o, 1:-1, 1:-1, c0:c0 + C_OUT].reshape(L.hw, C_OUT)
    return t[o, :, c0:c0 + C_OUT]


def _query(L: ReadLaunch, o: int) -> torch.Tensor:
    qk = L.args["qk"]
    return qk[L.qset[o]] if qk.dim() == 3 else qk


def _rerun(L: ReadLaunch, **over):
    A = dict(L.args)
    A["out"] = L.out.clone()
    A.update(over)
    return L.fn(**A)


def _same_bits(L: ReadLaunch, got: torch.Tensor, what: str) -> None:
    for a, b in zip(read_windows(L, L.out), read_windows(L, got)):
        if not torch.equal(a, b):
            d = (a.double() - b.double()).abs()
            raise AssertionError(f"{L.tag}: {what} differs from the production read (max |diff| {float(d.max()):.3g}, "
                                 f"{int((d > 0).sum())} elements)")


def tf32_stats(L: ReadLaunch, ws: torch.Tensor) -> Optional[list]:
    """mivos_memory_read_stats of the read that last ran in ws: [candidates, max per query, fallback queries,
    splits], or None where the call does not accept the launch."""
    from mivos_b200 import _lib
    st = (C.c_int64 * 4)()
    rc = _lib.lib().mivos_memory_read_stats(C.c_void_p(ws.data_ptr()), L.maps, int(L.args["slots"]), L.hw, L.top_k, st)
    return list(st) if rc == 0 else None


def _check_topk(L: ReadLaunch, idx: torch.Tensor, rows: torch.Tensor):
    """Checks 2 and 3 of a top-k / wide read over the queries `rows`: (worst err/bound, tie queries, tie swaps)."""
    out, bk, bv, k = L.out, L.args["bank_k"], L.args["bank_v"], L.top_k
    errs, refs, ties, swaps = [], [], 0, 0
    for o in range(L.maps):
        if L.qset[o] < 0:
            continue
        n = L.live[o]
        where = f"{L.tag}: object {o} (query set {L.qset[o]}, live {n})"
        assert n >= k, f"{where}: fewer live slots than top_k"
        q = scaled_q(_query(L, o)[rows.to(bk.device)])
        ko, vo = bk[o, :n].double(), bv[o, :n]
        got_o = map_rows(L, out, o)[rows.to(out.device)]
        chunk = max(1, min((1 << 25) // n, (1 << 24) // (k * C_OUT)))
        for c0 in range(0, rows.numel(), chunk):
            qc = q[c0:c0 + chunk]
            S = ko @ qc.t()                                             # [n, c]
            ic = idx[o, rows[c0:c0 + chunk].to(idx.device)].to(S.device).long()  # [c, k]
            bad = (ic < 0) | (ic >= n)
            if bool(bad.any()):
                qi = int(rows[c0 + int(bad.any(1).nonzero()[0, 0])])
                raise AssertionError(f"{where}: query {qi} selected a slot outside [0, {n})")
            srt = ic.sort(1).values
            dup = (srt[:, 1:] == srt[:, :-1]).any(1)
            if bool(dup.any()):
                raise AssertionError(f"{where}: query {int(rows[c0 + int(dup.nonzero()[0, 0])])} selected a slot twice")
            top = S.topk(min(k + 1, n), dim=0)
            kth = top.values[k - 1]
            gap = kth - top.values[k] if n > k else torch.full_like(kth, math.inf)
            same = (top.indices[:k].t().sort(1).values == srt).all(1)
            miss = ~same & (gap > TIE_EPS)
            if bool(miss.any()):
                j = int(miss.nonzero()[0, 0])
                raise AssertionError(f"{where}: query {int(rows[c0 + j])} selected another top-{k} set than float64 "
                                     f"with a k-th/(k+1)-th gap of {float(gap[j]):.3g} > TIE_EPS; "
                                     f"{int(miss.sum())} queries of this chunk")
            ties += int((gap <= TIE_EPS).sum())
            swaps += int((~same).sum())
            chosen = S.t().gather(1, ic)                               # [c, k]
            low = chosen.amin(1) < kth - TIE_EPS
            if bool(low.any()):
                j = int(low.nonzero()[0, 0])
                raise AssertionError(f"{where}: query {int(rows[c0 + j])} chose a slot of score "
                                     f"{float(chosen[j].min()):.8g} below the float64 k-th score "
                                     f"{float(kth[j]):.8g} - TIE_EPS")
            w = torch.softmax(chosen, 1)
            ref = torch.einsum("ck,ckd->cd", w, vo[ic.to(vo.device)].to(w.device).double())
            errs.append((got_o[c0:c0 + chunk].to(ref.device).double() - ref).abs())
            refs.append(ref)
    if not refs:
        return 0.0, ties, swaps
    err, ref = torch.cat(errs), torch.cat(refs)
    bound = RANGE_TERM * float(ref.abs().max()) + (ROUND_TERM * ref.abs() if L.out.dtype == torch.float16 else 0.0)
    ratio = err / (bound + 1e-300) if torch.is_tensor(bound) else err / max(bound, 1e-300)
    worst = float(ratio.max())
    if worst > 1.0:
        raise AssertionError(f"{L.tag}: read-out exceeds the bound {worst:.3g}x over the kernel's own top-{k} sets "
                             f"({int((ratio > 1).sum())} elements over)")
    return worst, ties, swaps


def _check_dense(L: ReadLaunch) -> float:
    from test_gpu_memread_dense import reference
    worst = 0.0
    bk, bv = L.args["bank_k"], L.args["bank_v"]
    for o in range(L.maps):
        if L.qset[o] < 0:
            continue
        ref, bound = reference(bk[o], bv[o], L.live[o], _query(L, o))
        if L.out.dtype == torch.float16:
            bound = bound + ROUND_TERM * ref.abs()
        r = float(((map_rows(L, L.out, o).double() - ref).abs() / bound).max())
        if r > 1.0:
            raise AssertionError(f"{L.tag}: object {o} (live {L.live[o]}) exceeds the dense read's bound {r:.3g}x")
        worst = max(worst, r)
    return worst


def check_read(L: ReadLaunch, *, max_scores: float = SAMPLE_SCORES, seed: int = 0) -> dict:
    """All checks of the read L, which has run (L.before: its output allocation before).  Raises AssertionError
    naming the launch and the worst query; returns the record of the table."""
    out = L.out
    changed_outside(L.before, out, lambda t: read_windows(L, t), f"{L.tag}: out",
                    lambda e: f"map {e // (out[0].numel())}, element {e % out[0].numel()} of the map")
    for win in read_windows(L, out):
        assert bool(torch.isfinite(win).all()), f"{L.tag}: read-out not finite"
    stats, sampled, ties, swaps, nq = None, False, 0, 0, L.hw
    if L.kind == "dense":
        worst = _check_dense(L)
    else:
        cuda = out.is_cuda
        ws = None
        if cuda and L.kind == "topk":
            from mivos_b200 import ops
            ws = torch.zeros(ops.memory_read_workspace_bytes(L.maps, int(L.args["slots"]), L.hw, L.top_k),
                             dtype=torch.uint8, device=out.device)
        got, idx, _ = _rerun(L, want_topk=True, workspace=ws)
        if cuda:
            torch.cuda.synchronize()
        _same_bits(L, got, "the want_topk re-run")
        if ws is not None:
            stats = tf32_stats(L, ws)
        if L.kind == "topk":
            from mivos_b200 import ops
            _same_bits(L, _rerun(L, algo=ops.MEMREAD_EXACT_SIMT, workspace=None), "the MEMREAD_EXACT_SIMT re-run")
        sampled = float(sum(L.live)) * L.hw > max_scores
        rows = sample_queries(L.hw, seed) if sampled else torch.arange(L.hw)
        nq = int(rows.numel())
        worst, ties, swaps = _check_topk(L, idx, rows)
    parts = sum(1 for s in L.qset if s >= 0)
    return dict(form=L.form, kind=L.kind, layout=L.layout, maps=L.maps, parts=parts, hw=L.hw, cap=L.cap,
                top_k=L.top_k, f16=out.dtype == torch.float16, q_div=L.q_div, counts=L.counts, first=L.first,
                live=tuple(L.live), bank0=L.args["bank_k"].storage_offset() // max(1, L.args["bank_k"][0].numel()),
                device_count=L.layout != "scalar" or L.args.get("dyn_slots") is not None,
                sampled=sampled, queries=nq, ties=ties, swaps=swaps, ratio=worst, stats=stats)


def checked_read(form: str, fn, A: dict, **kw) -> dict:
    """Snapshot, run and check one read launch (no synchronisation: CPU callers and Census._read, which
    synchronises around it)."""
    L = read_launch(form, fn, A)
    L.before = storage_bytes(L.out).clone()
    fn(**A)
    return check_read(L, **kw)


# ------------------------------------------------------------------ bank writes
@dataclass
class WriteLaunch:
    form: str
    args: dict
    maps: int
    hw: int
    cap: int
    groups: list               # (first map, end map, frame) per group / set
    t_max: int
    first: Optional[tuple]
    before: list = field(default_factory=list)

    @property
    def sig(self) -> tuple:
        return (self.form, self.maps, self.hw, self.cap, tuple(g[2] for g in self.groups), self.first, self.t_max)

    @property
    def tag(self) -> str:
        return f"{self.form} (maps {self.maps}, hw {self.hw}, cap {self.cap}, groups {self.groups}, t_max {self.t_max})"


def write_launch(form: str, A: dict) -> WriteLaunch:
    layout = WRITES[form]
    bk = A["bank_k"]
    hw = A["h"] * A["w"]
    first = None
    if layout == "scalar":
        t = _ints(A["dyn_t"])[0] if A.get("dyn_t") is not None else int(A["t"])
        groups, t_max, maps = [(0, A["k"], t)], int(A["t"]), A["k"]
    elif layout == "sets":
        per = A["k"] // A["sets"]
        ts = _ints(A["dyn_t"])[:A["sets"]]
        groups, t_max, maps = [(s * per, (s + 1) * per, ts[s]) for s in range(A["sets"])], int(A["t_max"]), A["k"]
    else:
        first = tuple(_ints(A["first"]))
        ts = _ints(A["dyn_t"])[:len(first) - 1]
        maps = A["n"]
        groups = [(max(first[g], 0), min(first[g + 1], maps), ts[g]) for g in range(len(first) - 1)]
        t_max = int(A["t_max"])
    return WriteLaunch(form, A, maps, hw, bk.shape[1], groups, t_max, first)


def write_bytes(A: dict) -> int:
    return A["bank_k"].untyped_storage().nbytes() + A["bank_v"].untyped_storage().nbytes()


def check_write(L: WriteLaunch) -> dict:
    A = L.args
    halo, hw = A["halo"], L.hw
    for name, coff, c, before in (("bank_k", A["coff_k"], 128, L.before[0]), ("bank_v", A["coff_v"], 512, L.before[1])):
        bank = A[name]
        exp = before.clone()
        view = like(exp, bank)
        for a, b, t in L.groups:
            if a < b and 0 <= t <= L.t_max:
                view[a:b, t * hw:(t + 1) * hw] = halo[a:b, 1:-1, 1:-1, coff:coff + c].reshape(b - a, hw, c)
        diff = (exp != storage_bytes(bank)).nonzero()
        if diff.numel():
            e = int(diff[0, 0]) // 4 - bank.storage_offset()
            per_map = bank.shape[1] * c
            if 0 <= e < bank.numel():
                m, slot = e // per_map, e % per_map // c
                g = [i for i, (a, b, _t) in enumerate(L.groups) if a <= m < b]
                loc = (f"map {m} (group {g[0] if g else None}, frame {L.groups[g[0]][2] if g else None}), slot {slot} "
                       f"(frame {slot // hw}), channel {e % c}")
            else:
                loc = f"byte {int(diff[0, 0])} of the allocation, outside the view"
            raise AssertionError(f"{L.tag}: {name} differs from the expected write: {diff.shape[0]} bytes, first at "
                                 f"{loc}")
    return dict(form=L.form, maps=L.maps, hw=hw, cap=L.cap, groups=len(L.groups), frames=tuple(g[2] for g in L.groups),
                t_max=L.t_max, first=L.first)


def checked_write(form: str, fn, A: dict) -> dict:
    L = write_launch(form, A)
    L.before = [storage_bytes(A["bank_k"]).clone(), storage_bytes(A["bank_v"]).clone()]
    fn(**A)
    return check_write(L)


# ------------------------------------------------------------------ the recorder
class MemoryCensus:
    """Recorder of memory reads and bank writes; `record(s)` checks every eager launch of scenario s."""

    def __init__(self, max_scores: float = SAMPLE_SCORES, max_bank_bytes: int = BANK_SNAPSHOT_BYTES):
        self.max_scores, self.max_bank_bytes = max_scores, max_bank_bytes
        self.records = []
        self.writes = []
        self.seen = Counter()
        self.checked = Counter()
        self.captured = Counter()
        self.too_big = Counter()
        self._sigs = set()

    @contextlib.contextmanager
    def record(self, scenario: str):
        from mivos_b200 import ops
        saved = {name: getattr(ops, name) for name in list(READS) + list(WRITES)}
        for name, fn in saved.items():
            setattr(ops, name, self._wrap(scenario, name, fn))
        try:
            yield self
        finally:
            for name, fn in saved.items():
                setattr(ops, name, fn)

    def _wrap(self, scenario, form, fn):
        def launch(*args, **kw):
            return self._launch(scenario, form, fn, args, kw)
        return launch

    def _launch(self, scenario, form, fn, args, kw):
        A = bind(fn, args, kw)
        cuda = A["bank_k"].is_cuda
        if cuda and torch.cuda.is_current_stream_capturing():
            self.captured[scenario] += 1
            return fn(*args, **kw)
        self.seen[scenario] += 1
        if cuda:
            torch.cuda.synchronize()
        L = read_launch(form, fn, A) if form in READS else write_launch(form, A)
        if L.sig in self._sigs:
            return fn(*args, **kw)
        if form in WRITES and write_bytes(A) > self.max_bank_bytes:
            self.too_big[scenario] += 1
            return fn(*args, **kw)
        self._sigs.add(L.sig)
        if form in READS:
            L.before = storage_bytes(L.out).clone()
        else:
            L.before = [storage_bytes(A["bank_k"]).clone(), storage_bytes(A["bank_v"]).clone()]
        res = fn(*args, **kw)
        if cuda:
            from mivos_b200 import _lib
            torch.cuda.synchronize()
            _lib.poll_kernel_error()
        if form in READS:
            rec = check_read(L, max_scores=self.max_scores, seed=len(self.records))
            self.records.append(dict(rec, scenario=scenario))
        else:
            self.writes.append(dict(check_write(L), scenario=scenario))
        self.checked[scenario] += 1
        del L
        return res

    def table(self) -> str:
        def short(t):
            s = "-" if t is None else ",".join(str(v) for v in t)
            return s if len(s) <= 22 else s[:19] + "..."
        lines = [f"{'scenario':20s} {'form':24s} {'K':>3s} {'hw':>5s} {'cap':>6s} {'k':>4s} {'cat':3s} {'qd':>2s} "
                 f"{'counts':22s} {'first':22s} {'queries':>8s} {'ties':>5s} {'err/bound':>9s} {'fallback':>9s}"]
        for r in self.records:
            st = r["stats"]
            fb = f"{st[2]}/{r['maps'] * r['hw']}" if st else "-"
            lines.append(f"{r['scenario']:20s} {r['form']:24s} {r['maps']:3d} {r['hw']:5d} {r['cap']:6d} "
                         f"{r['top_k'] or 0:4d} {'f16' if r['f16'] else 'f32':3s} {r['q_div']:2d} "
                         f"{short(r['counts']):22s} {short(r['first']):22s} {r['queries']:8d}"
                         f"{'*' if r['sampled'] else ' '}{r['ties']:5d} {r['ratio']:9.3g} {fb:>9s}")
        for r in self.writes:
            lines.append(f"{r['scenario']:20s} {r['form']:24s} {r['maps']:3d} {r['hw']:5d} {r['cap']:6d} "
                         f"frames {short(r['frames'])} t_max {r['t_max']} first {short(r['first'])}: bit-exact")
        return "\n".join(lines)

    def summary(self) -> str:
        out = []
        for s in self.seen:
            rs = [r for r in self.records if r["scenario"] == s]
            st = [r["stats"] for r in rs if r["stats"]]
            q = sum(r["maps"] * r["hw"] for r in rs if r["stats"])
            fb = f"{sum(x[2] for x in st)}/{q} queries on the exact fallback" if st else "no TF32-path reads"
            out.append(f"{s}: {self.seen[s]} memory launches seen, {self.checked[s]} checked "
                       f"({len(rs)} reads, {sum(1 for w in self.writes if w['scenario'] == s)} bank writes, "
                       f"{self.too_big[s]} bank writes above the snapshot limit), worst read err/bound "
                       f"{max((r['ratio'] for r in rs), default=0.0):.3g}; {fb}")
        return "\n".join(out)
