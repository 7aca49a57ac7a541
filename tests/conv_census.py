"""TEST INFRASTRUCTURE: the conv census — every mivos_conv_gemm launch of a real session, checked on its own operands
against a float64 restatement of the ABI contract in include/mivos_b200.h:

    y[r, co] = bias[co] + sum_t sum_ci A[r + off(t), ci] * W[t, co, ci]  (+ residual[r, res_coff + co])  (relu)

for the interior rows r of the output map, with off(t) = (t/3 - 1)(w+2) + (t%3 - 1) for 9 taps, (t - 2)(w+2) for 4
and 0 for 1; rows outside the operand matrix read 0 (the TMA zero fill).  A is what the tensor core multiplies (fp16
values, or fp32 truncated to TF32), W the packed, already-rounded weights, the residual its stored value.

Checks per launch (DESIGN.md section 6):
  1. |got - y| <= 2e-5 max|y| + 2^-23 (taps cin_pad / k_mma + 10) (|bias| + sum|a w| + |residual|) + 2^-11 |y|:
     accumulation order relative to the output range, plus one fp32 ulp per accumulator update (k_mma = 8 TF32 /
     16 fp16 products per MMA instruction) of the element's own magnitude sum — long K over operands that cancel
     (the 9216-long key/value projection) exceeds the first term alone —, plus, for fp16 and round_tf32 outputs, one
     rounding of the result; round_tf32 outputs also have zero low 13 bits;
  2. every byte of the allocations out / out_relu live in, outside [interior rows] x [coff, coff + cout) of the
     launch's n maps, keeps its value: the HALO border, channels past cout, the neighbouring windows of concat maps,
     and the maps of the allocation outside the view (the next object chunk of a logits map sliced lg[k0:k0 + n],
     the clips past a lock-step tick's prefix);
  3. out_relu == relu(out) on the window;
  4. the premises of the zero padding: the operand's HALO border rows are zero in the read window (9 and 4 taps), the
     packed weights are zero past the real K, and the operand is finite everywhere it is read;
  5. the outputs are finite.
Check 1 compares every interior row, or, above SAMPLE_MACS multiply-adds, a deterministic sample (`sample_rows`).

`Census.record(scenario)` replaces mivos_b200.ops.conv_gemm — every engine launches through engine._cg — so that each
eager launch is synchronised, snapshotted, run, polled for a kernel error and checked before the session goes on.
Launches are deduplicated by signature (layer, shape, types, windows, residual / dual output, plan): the first is
checked, the rest are counted.  The plan is (BN, S, CTAs): tile width and split-K factor from mivos_conv_plan, CTAs
per SM from mivos_conv_plan_residency.  Device-agnostic and importable without a GPU: tests/test_conv_census_cpu.py drives
`check_launch` with emulated kernels (tests/abi_emulator.py) and mutations of them."""
from __future__ import annotations

import contextlib
import ctypes as C
from collections import Counter
from dataclasses import dataclass
from typing import Optional

import torch

TF32_LOW = 0x1FFF
RANGE_TERM = 2e-5          # of max|y|: fp32 accumulation order
ROUND_TERM = 2.0 ** -11    # of |y|: one rounding of an fp16 or round_tf32 output
ACC_UNIT = 2.0 ** -23      # of |bias| + sum|a*w| (+ |residual|), per accumulator update: one fp32 ulp
SAMPLE_MACS = 1e10         # rows x taps x cin_pad x cout_pad above which check 1 samples rows
SAMPLE_RANDOM = 16384
BM = 128                   # rows per M tile of the kernel


def operand64(t: torch.Tensor) -> torch.Tensor:
    """What the tensor core multiplies, in float64: fp16 values, or fp32 truncated to TF32."""
    if t.dtype == torch.float16:
        return t.double()
    return (t.contiguous().view(torch.int32) & ~TF32_LOW).view(torch.float32).double()


def tap_offsets(taps: int, w: int):
    if taps == 9:
        return [(t // 3 - 1) * (w + 2) + (t % 3 - 1) for t in range(9)]
    if taps == 4:
        return [(t - 2) * (w + 2) for t in range(4)]
    assert taps == 1, taps
    return [0]


def real_k(pc) -> int:
    """Columns of a packed tap that hold weights; the rest of cin_pad must be zero."""
    if pc.taps == 9:
        return pc.cin
    if pc.taps == 4:  # space-to-depth stem: 2 x 4 x 2 x cin
        return 16 * pc.cin
    return pc.ksize * pc.ksize * pc.cin  # 1x1, or a pre-gathered (ky, kx, ci) matrix


def interior_mask(rows: torch.Tensor, n: int, h: int, w: int) -> torch.Tensor:
    img = rows % ((h + 2) * (w + 2))
    line, col = img // (w + 2), img % (w + 2)
    return (rows >= 0) & (rows < n * (h + 2) * (w + 2)) & (line >= 1) & (line <= h) & (col >= 1) & (col <= w)


def interior_rows(n: int, h: int, w: int, device) -> torch.Tensor:
    line = torch.arange(1, h + 1, device=device)[:, None] * (w + 2) + torch.arange(1, w + 1, device=device)[None, :]
    return (torch.arange(n, device=device)[:, None] * ((h + 2) * (w + 2)) + line.reshape(1, -1)).reshape(-1)


def sample_rows(n: int, h: int, w: int, device, seed: int = 0) -> torch.Tensor:
    """Every row of the first two and last two 128-row tiles; rows m0, m0+63, m0+64, m0+127 of every tile; the first
    and last interior line of each image; SAMPLE_RANDOM seeded random interior rows.  Interior rows only, sorted."""
    rows = n * (h + 2) * (w + 2)
    tiles = (rows + BM - 1) // BM
    ends = [t for t in (0, 1, tiles - 2, tiles - 1) if 0 <= t < tiles]
    parts = [torch.arange(t * BM, (t + 1) * BM) for t in sorted(set(ends))]
    m0 = torch.arange(tiles) * BM
    parts += [m0 + d for d in (0, 63, 64, 127)]
    img = torch.arange(n)[:, None] * ((h + 2) * (w + 2)) + torch.arange(1, w + 1)[None, :]
    parts += [(img + (w + 2)).reshape(-1), (img + h * (w + 2)).reshape(-1)]
    g = torch.Generator().manual_seed(seed)
    k = torch.randint(0, n * h * w, (SAMPLE_RANDOM,), generator=g)
    parts.append((k // (h * w)) * ((h + 2) * (w + 2)) + ((k % (h * w)) // w + 1) * (w + 2) + k % w + 1)
    r = torch.cat(parts)
    return torch.unique(r[interior_mask(r, n, h, w)]).to(device)


def storage_bytes(t: torch.Tensor) -> torch.Tensor:
    """The whole allocation `t` lives in (its untyped storage), as a uint8 tensor sharing it."""
    return torch.empty(0, dtype=torch.uint8, device=t.device).set_(t.untyped_storage())


def like(buf: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    """A view of the byte buffer `buf` (a copy of t's allocation) with t's type, offset, shape and strides."""
    return torch.empty(0, dtype=t.dtype, device=buf.device).set_(buf.untyped_storage(), t.storage_offset(), t.size(),
                                                                  t.stride())


def changed_outside(before: torch.Tensor, t: torch.Tensor, windows, what: str, where=None) -> None:
    """Raise AssertionError if a byte of t's allocation other than windows(t) differs from `before` (the
    storage_bytes clone taken before the launch).  `windows(x)` lists the written views of a tensor x laid out as t;
    `where(e)` names the element at offset e of the view."""
    exp = before.clone()
    for a, b in zip(windows(like(exp, t)), windows(t)):
        a.copy_(b)
    diff = (exp != storage_bytes(t)).nonzero()
    if not diff.numel():
        return
    byte = int(diff[0, 0])
    e = byte // t.element_size() - t.storage_offset()
    if 0 <= e < t.numel() and t.is_contiguous():
        loc = where(e) if where else f"element {e} of the view"
    else:
        loc = f"byte {byte} of the allocation, outside the view of {tuple(t.shape)} at element offset {t.storage_offset()}"
    raise AssertionError(f"{what} written outside its window: {diff.shape[0]} bytes, first at {loc}")


@dataclass
class Launch:
    """One conv launch: its arguments and snapshots (clones) of what it reads and of its outputs before it ran."""

    layer: str
    pc: object
    n: int
    h: int
    w: int
    x: torch.Tensor                   # operand window [in_rows, cin_pad]
    res: Optional[torch.Tensor]       # residual window [rows, cout], stored type
    out: torch.Tensor                 # the allocation `out` lives in before the launch (bytes)
    out_coff: int
    out_relu: Optional[torch.Tensor]  # the allocation of the ReLU copy before the launch (bytes)
    out_relu_coff: int
    relu: bool
    rnd: bool                         # round_tf32 in effect (fp32 outputs only)
    plan: Optional[tuple]
    in_desc: str
    out_desc: str

    @property
    def rows(self) -> int:
        return self.n * (self.h + 2) * (self.w + 2)


def _win(t: torch.Tensor, coff: int, c: int) -> str:
    return f"{'f16' if t.dtype == torch.float16 else 'f32'}[{coff}:{coff + c}/{t.shape[-1]}]"


def snapshot(x, pc, n, h, w, out, *, in_coff=0, out_coff=0, relu=False, residual=None, res_coff=0, out_relu=None,
             out_relu_coff=0, round_tf32=False, splitk_ws=None, layer="?", plan=None) -> Launch:
    rows = n * (h + 2) * (w + 2)
    xw = x.reshape(-1, x.shape[-1])[:, in_coff:in_coff + pc.cin_pad].clone()
    res = None
    if residual is not None:
        res = residual.reshape(-1, residual.shape[-1])[:rows, res_coff:res_coff + pc.cout].clone()
    in_desc = _win(x, in_coff, pc.cin_pad) + ("" if x.dim() == 4 else " mat")
    out_desc = _win(out, out_coff, pc.cout)
    if residual is not None:
        out_desc += " +res" + _win(residual, res_coff, pc.cout)[3:]
    if out_relu is not None:
        out_desc += " dual" + _win(out_relu, out_relu_coff, pc.cout)[3:]
    return Launch(layer, pc, n, h, w, xw, res, storage_bytes(out).clone(), out_coff,
                  None if out_relu is None else storage_bytes(out_relu).clone(), out_relu_coff, bool(relu),
                  bool(round_tf32) and out.dtype == torch.float32, plan, in_desc, out_desc)


def reference(L: Launch, rows: torch.Tensor, with_abs: bool = False):
    """float64 y[rows, :cout] of the ABI contract, in row chunks; with_abs: also |bias| + sum |a*w| (+ |residual|)."""
    pc = L.pc
    in_rows = L.x.shape[0]
    W = pc.weight[:, :pc.cout, :].double()
    bias = pc.bias[:pc.cout].double()
    offs = tap_offsets(pc.taps, L.w)
    chunk = max(1024, (1 << 25) // pc.cin_pad)
    ys, ss = [], []
    for r in rows.split(chunk):
        acc = bias.expand(r.numel(), -1).clone()
        mag = bias.abs().expand(r.numel(), -1).clone() if with_abs else None
        for t, off in enumerate(offs):
            idx = r + off
            ok = (idx >= 0) & (idx < in_rows)
            a = operand64(L.x[idx.clamp(0, in_rows - 1)])
            a[~ok] = 0.0
            acc += a @ W[t].t()
            if with_abs:
                mag += a.abs() @ W[t].abs().t()
        if L.res is not None:
            acc += L.res[r].double()
            if with_abs:
                mag += L.res[r].double().abs()
        ys.append(acc.clamp_min_(0.0) if L.relu else acc)
        ss.append(mag)
    return (torch.cat(ys), torch.cat(ss)) if with_abs else torch.cat(ys)


def accumulation_steps(L: Launch) -> int:
    """fp32 accumulator updates of one output element: one per MMA instruction (K = 8 TF32 / 16 fp16 products,
    exact in fp32), plus the split-K partial sums, bias and residual (at most 8 splits + 2)."""
    return L.pc.taps * L.pc.cin_pad // (16 if L.x.dtype == torch.float16 else 8) + 10


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _where(L: Launch, row: int) -> str:
    p = (L.h + 2) * (L.w + 2)
    return f"row {row} (image {row // p}, line {row % p // (L.w + 2)}, col {row % p % (L.w + 2)})"


def _outside_changed(before, after, L: Launch, coff: int, what: str):
    C = after.shape[-1]
    changed_outside(before, after, lambda t: [window(t, L.n, L.h, L.w, coff, L.pc.cout)], what,
                    lambda e: f"{_where(L, e // C)} channel {e % C}")


def window(t: torch.Tensor, n: int, h: int, w: int, coff: int, cout: int) -> torch.Tensor:
    """The written window of a HALO output map: interior rows x channels [coff, coff + cout) (a view)."""
    rows = n * (h + 2) * (w + 2)
    return t.reshape(-1, t.shape[-1])[:rows].view(n, h + 2, w + 2, -1)[:, 1:-1, 1:-1, coff:coff + cout]


def check_premises(L: Launch) -> None:
    pc = L.pc
    rows = min(L.rows, L.x.shape[0])
    assert bool(torch.isfinite(L.x[:rows]).all()), f"{L.layer}: operand not finite where it is read"
    if pc.taps in (9, 4):
        xh = L.x[:L.rows].view(L.n, L.h + 2, L.w + 2, -1)
        border = torch.cat([xh[:, 0].reshape(-1), xh[:, -1].reshape(-1), xh[:, :, 0].reshape(-1), xh[:, :, -1].reshape(-1)])
        assert bool((border == 0).all()), f"{L.layer}: operand HALO border not zero in the read window"
    assert bool((pc.weight[:, :, real_k(pc):] == 0).all()), f"{L.layer}: packed weights not zero past K = {real_k(pc)}"


def macs(L: Launch) -> float:
    return float(L.rows) * L.pc.taps * L.pc.cin_pad * L.pc.cout_pad


def check_launch(L: Launch, out, out_relu=None, *, max_macs: float = SAMPLE_MACS, seed: int = 0) -> dict:
    """Checks 1-5 of the launch L, whose outputs are now `out` / `out_relu`.  Raises AssertionError with the layer,
    plan and worst element; returns the record of the table."""
    pc = L.pc
    tag = f"{L.layer} (n h w {L.n} {L.h} {L.w}, plan {L.plan})"
    check_premises(L)
    _outside_changed(L.out, out, L, L.out_coff, f"{tag}: out")
    win = window(out, L.n, L.h, L.w, L.out_coff, pc.cout)
    assert bool(torch.isfinite(win).all()), f"{tag}: output not finite"
    if L.out_relu is not None:
        _outside_changed(L.out_relu, out_relu, L, L.out_relu_coff, f"{tag}: out_relu")
        assert torch.equal(window(out_relu, L.n, L.h, L.w, L.out_relu_coff, pc.cout), win.clamp_min(0)), \
            f"{tag}: out_relu != relu(out)"
    if L.rnd:
        low = int((_bits(win) & TF32_LOW).abs().max()) if win.numel() else 0
        assert low == 0, f"{tag}: round_tf32 output has nonzero low 13 bits"
    sampled = macs(L) > max_macs
    rows = sample_rows(L.n, L.h, L.w, L.x.device, seed) if sampled else interior_rows(L.n, L.h, L.w, L.x.device)
    y, mag = reference(L, rows, with_abs=True)
    got = out.reshape(-1, out.shape[-1])[rows, L.out_coff:L.out_coff + pc.cout].double()
    rounded = L.rnd or out.dtype == torch.float16
    bound = RANGE_TERM * float(y.abs().max()) + ACC_UNIT * accumulation_steps(L) * mag
    if rounded:
        bound = bound + ROUND_TERM * y.abs()
    err = (got - y).abs()
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if worst > 1.0:
        i = int(ratio.argmax())
        r, c = int(rows[i // pc.cout]), i % pc.cout
        raise AssertionError(f"{tag}: |got - y| exceeds the bound {worst:.3g}x at {_where(L, r)} channel {c}: got "
                             f"{float(got.reshape(-1)[i])!r}, float64 {float(y.reshape(-1)[i])!r}, max|y| "
                             f"{float(y.abs().max()):.4g}; {int((ratio > 1).sum())} elements over")
    bn, sp, ctas = L.plan if L.plan else (0, 0, 0)
    map_bytes = (L.h + 2) * (L.w + 2) * out.shape[-1] * out.element_size()
    return dict(layer=L.layer, nhw=f"{L.n}x{L.h}x{L.w}", taps=pc.taps, cin_pad=pc.cin_pad, cout=pc.cout,
                inp=L.in_desc, outp=L.out_desc, bn=bn, s=sp, ctas=ctas, rows=int(rows.numel()), sampled=sampled,
                ratio=worst, alloc_maps=L.out.numel() // map_bytes,
                n=L.n, f16=L.x.dtype == torch.float16, out_f16=out.dtype == torch.float16, res=L.res is not None,
                dual=L.out_relu is not None, out_coff=L.out_coff, mat=L.in_desc.endswith("mat"))


def conv_plan(x, pc, n, h, w, out, kw, sms: int = 0):
    """(BN, S, CTAs per SM) that mivos_conv_plan and mivos_conv_plan_residency report for the argument block
    ops.conv_gemm builds from these arguments."""
    from mivos_b200 import _lib, ops
    a = ops.conv_args(x, pc, n, h, w, out, **kw)
    bn, sp, ctas = C.c_int(0), C.c_int(0), C.c_int(0)
    lib = _lib.load()
    _lib.check(lib.mivos_conv_plan(C.byref(a), sms, C.byref(bn), C.byref(sp)), "mivos_conv_plan")
    _lib.check(lib.mivos_conv_plan_residency(C.byref(a), sms, C.byref(ctas)), "mivos_conv_plan_residency")
    return bn.value, sp.value, ctas.value


class Census:
    """Recorder of conv launches.  `label(pcs)` names the PackedConvs of an engine (its `pc` dict); `record(s)`
    checks every eager launch of scenario s while the context is open."""

    def __init__(self, max_macs: float = SAMPLE_MACS, sms: int = 0):
        self.max_macs, self.sms = max_macs, sms
        self.names = {}
        self.records = []
        self.seen = Counter()
        self.checked = Counter()
        self.captured = Counter()
        self._sigs = set()

    def label(self, pcs: dict, prefix: str = "") -> None:
        for k, v in pcs.items():
            self.names[id(v)] = (prefix + k, v)  # keeps v alive, so that its id stays its own

    @contextlib.contextmanager
    def record(self, scenario: str):
        from mivos_b200 import ops
        launch = ops.conv_gemm

        def conv_gemm(x, pc, n, h, w, out, **kw):
            return self._launch(launch, scenario, x, pc, n, h, w, out, kw)
        ops.conv_gemm = conv_gemm
        try:
            yield self
        finally:
            ops.conv_gemm = launch

    def _launch(self, launch, scenario, x, pc, n, h, w, out, kw):
        cuda = x.is_cuda
        if cuda and torch.cuda.is_current_stream_capturing():
            self.captured[scenario] += 1
            return launch(x, pc, n, h, w, out, **kw)
        self.seen[scenario] += 1
        layer = self.names.get(id(pc), ("?",))[0]
        plan = conv_plan(x, pc, n, h, w, out, kw, self.sms) if cuda else None
        res, dual = kw.get("residual"), kw.get("out_relu")
        sig = (layer, pc.taps, pc.cin_pad, pc.cout, n, h, w, x.dtype, x.shape[-1], x.dim(), kw.get("in_coff", 0),
               out.dtype, out.shape[-1], kw.get("out_coff", 0), bool(kw.get("relu")), bool(kw.get("round_tf32")),
               None if res is None else (res.shape[-1], kw.get("res_coff", 0)),
               None if dual is None else (dual.shape[-1], kw.get("out_relu_coff", 0)), plan)
        if sig in self._sigs:
            return launch(x, pc, n, h, w, out, **kw)
        self._sigs.add(sig)
        if cuda:
            torch.cuda.synchronize()
        L = snapshot(x, pc, n, h, w, out, layer=layer, plan=plan, **kw)
        launch(x, pc, n, h, w, out, **kw)
        if cuda:
            from mivos_b200 import _lib
            torch.cuda.synchronize()
            _lib.poll_kernel_error()
        rec = check_launch(L, out, dual, max_macs=self.max_macs, seed=len(self.records))
        rec["scenario"] = scenario
        self.records.append(rec)
        self.checked[scenario] += 1
        del L
        return out

    def table(self) -> str:
        head = (f"{'scenario':24s} {'layer':44s} {'n x h x w':>13s} {'taps':>4s} {'cin_p':>5s} {'cout':>4s} "
                f"{'in':24s} {'out':44s} {'BN':>3s} {'S':>2s} {'CTA':>3s} {'rows':>8s} {'err/bound':>9s}")
        lines = [head]
        for r in self.records:
            lines.append(f"{r['scenario']:24s} {r['layer']:44s} {r['nhw']:>13s} {r['taps']:4d} {r['cin_pad']:5d} "
                         f"{r['cout']:4d} {r['inp']:24s} {r['outp']:44s} {r['bn']:3d} {r['s']:2d} {r['ctas']:3d} "
                         f"{r['rows']:8d}{'*' if r['sampled'] else ' '}{r['ratio']:9.3g}")
        return "\n".join(lines)

    def summary(self) -> str:
        out = []
        for s in self.seen:
            rs = [r["ratio"] for r in self.records if r["scenario"] == s]
            out.append(f"{s}: {self.seen[s]} launches seen, {self.checked[s]} checked, worst err/bound "
                       f"{max(rs) if rs else 0.0:.3g}")
        return "\n".join(out)
