"""TEST INFRASTRUCTURE: the operator census — every launch of the non-GEMM operators a real session makes (stem
gathers, layout copies, the decoder's skip-adds, the aggregation, argmax, attention, the S2M resizes and pooling, the
table stores), checked on its own operands against float64 restatements of include/mivos_b200.h, with the
references and elementwise bounds of tests/op_references.py (the ones the ragged-shape tests use).

Per launch (DESIGN.md section 6):
  1. the output window holds the reference: bit for bit for copies, gathers, pooling, argmax, padding, the frame
     normalisation (the kernel's fp32 operations are the header expression's, in its order) and table stores; within
     the operator's bound otherwise, plus one rounding (2^-11 |ref|) into fp16 maps.  The aggregation is checked
     against aggregate_reference of the kernel's own fp32 `raw` (re-run into scratch when production does not ask for
     it: the prob bits must not change), the hard aggregation as a one-hot within K e^-19 where the fp64 hard-logit
     gap exceeds 20.  "Others" of stem_gather_range sums over all K masks, of stem_gather_groups over the group;
  2. every value in the window is finite;
  3. no byte of the whole allocation of any output changes outside its window (conv_census.changed_outside): the HALO
     border, other channels, maps no group holds, maps past a lock-step tick's prefix, the next object chunk.  Each
     output of a launch with several (raw_out + prob_out, masks_padded + masks_out, x + x_relu) is checked on its own;
     x_relu is also relu(x) bit for bit.
Allocations above SNAPSHOT_BYTES are counted, not checked.

`OpCensus.record(scenario)` replaces the leaf attributes of mivos_b200.ops named in FORMS (the functions that call a
mivos_* launch symbol); aggregate_any, upsample4x_sigmoid_aggregate_any and attention_op look their leaves up at call
time, so their calls are caught too.  Stream-captured launches pass through.  Launches are deduplicated by signature:
the form, every tensor operand's shape, type, allocation size and offset, the scalar arguments (windows, flags,
prefix counts) and the contents of the group table.  Device-agnostic and importable without a GPU:
tests/test_op_census_cpu.py drives `checked` with emulated kernels and their mutations."""
from __future__ import annotations

import contextlib
import inspect
import math
from collections import Counter

import torch
import torch.nn.functional as F

import op_references as R
from conv_census import changed_outside, storage_bytes

SNAPSHOT_BYTES = 2 << 30     # output allocations above this are counted, not checked (the 1088p S2M matrices fit)
HARD_GAP = 20.0              # fp64 hard-logit gap above which the hard aggregation is one-hot
NORM_MEAN = (0.485, 0.456, 0.406)  # include/mivos_b200.h, mivos_frames_u8_normalize
NORM_STD = (0.229, 0.224, 0.225)

# The leaves of the memory and conv censuses, and the ABI entry points none of the three censuses check, with why.
CONV_FORMS = ("conv_gemm",)
NOT_CENSUSED = {
    "mivos_abi_version": "no kernel launch: the ABI version",
    "mivos_last_error": "no kernel launch: the error string",
    "mivos_check_device": "no kernel launch: the device check",
    "mivos_poll_kernel_error": "no kernel launch: reads the kernel error word",
    "mivos_launch_count": "no kernel launch: the launch counter",
    "mivos_add_launch_count": "no kernel launch: the launch counter",
    "mivos_host_register": "no kernel launch: page-locks host memory",
    "mivos_host_unregister": "no kernel launch: unpins host memory",
    "mivos_conv_tile_override": "no kernel launch: an override knob of the conv plan",
    "mivos_conv_plan": "no kernel launch: the conv plan",
    "mivos_conv_plan_residency": "no kernel launch: the conv plan",
    "mivos_conv_residency_override": "no kernel launch: an override knob of the conv plan",
    "mivos_memory_read_workspace": "no kernel launch: a workspace size",
    "mivos_memory_read_dense_workspace": "no kernel launch: a workspace size",
    "mivos_memory_read_wide_workspace": "no kernel launch: a workspace size",
    "mivos_memory_read_stats": "no kernel launch: reads the statistics of a workspace",
    "mivos_attention_plan": "no kernel launch: the attention plan",
    "mivos_stem_frames_plan": "no kernel launch: the stem gather plan",
    "mivos_store_i32": "not launched by the package (store_words replaced it)",
}
NOT_CENSUSED_REASONS = ("no kernel launch", "not launched by the package")


def _sym(t):
    return "f16" if t.dtype == torch.float16 else "f32" if t.dtype == torch.float32 else str(t.dtype)[6:]


def bind(fn, args, kw) -> dict:
    b = inspect.signature(fn).bind(*args, **kw)
    b.apply_defaults()
    return dict(b.arguments)


def _ints(t) -> list:
    return [int(v) for v in t.reshape(-1).cpu().tolist()]


def groups_of(first: list, maps: int) -> list:
    """(g, a, b) of every group that takes part: 0 <= a < b <= maps (include/mivos_b200.h, object-group forms)."""
    return [(g, a, b) for g, (a, b) in enumerate(zip(first, first[1:])) if 0 <= a < b <= maps]


def interior(t, n, h, w, coff, c):
    """Interior pixels x channels [coff, coff + c) of the first n maps of a HALO map (a view)."""
    return t[:n, 1:h + 1, 1:w + 1, coff:coff + c]


def nchw(t):
    return t.permute(0, 3, 1, 2).double()


def matrix_rows(t, n, h, w, c0, c1):
    """Rows of the first n HALO images (h, w) of a gathered matrix, columns [c0, c1) (a view [n, h+2, w+2, c])."""
    rows = n * (h + 2) * (w + 2)
    return t.reshape(-1, t.shape[-1])[:rows].view(n, h + 2, w + 2, -1)[..., c0:c1]


def flat(t, n):
    return t.reshape(-1)[:n]


class Mismatch(AssertionError):
    pass


def exact(what, got, ref):
    ref = ref.to(got.device).to(got.dtype)
    if not torch.equal(got, ref):
        d = got != ref
        i = int(d.reshape(-1).nonzero()[0, 0])
        raise Mismatch(f"{what}: not bit-exact at {int(d.sum())} of {got.numel()} elements, first at flat index {i}: "
                       f"got {float(got.reshape(-1)[i])!r}, expected {float(ref.reshape(-1)[i])!r}")
    return 0.0


def bounded(what, got, ref, bound):
    """max |got - ref| / bound over the elements (0/0 counts as 0, x/0 as inf); raises above 1."""
    got = got.to(ref.device).double()
    err = (got - ref).abs()
    if not torch.is_tensor(bound):
        bound = torch.full_like(ref, float(bound))
    bound = bound.to(ref.device).expand_as(err)
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    ratio = torch.where(torch.isnan(err), math.inf, ratio)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if worst > 1.0:
        i = int(ratio.reshape(-1).argmax())
        raise Mismatch(f"{what}: |got - ref| exceeds the bound {worst:.3g}x at flat index {i}: got "
                       f"{float(got.reshape(-1)[i])!r}, float64 {float(ref.reshape(-1)[i])!r}, bound "
                       f"{float(bound.reshape(-1)[i]):.3g}; {int((ratio > 1).sum())} elements over")
    return worst


def r16(bound, ref, dtype):
    return R.round16(bound, ref, dtype)


# ------------------------------------------------------------------ the forms
# Each form: spec(A) -> {output argument: windows(t) -> list of written views} (None: the launch allocates it and
# returns it), and check(A0, O, fn) -> (worst err/bound, facts) with A0 the operands as they were before the launch
# and O the outputs after it.
# A form whose operands are raw addresses also has pre(A, hosts) -> state, taken before the launch (A0["_pre"]).
class Form:
    def __init__(self, spec, check, returns=None, pre=None):
        self.spec, self.check, self.returns, self.pre = spec, check, returns, pre


FORMS = {}


def form(name, returns=None):
    def deco(pair):
        parts = pair()
        FORMS[name] = Form(parts[0], parts[1], returns, *parts[2:])
        return pair
    return deco


def _synced(t):
    """Synchronise and poll the kernel error after a re-run on the device."""
    if t.is_cuda:
        from mivos_b200 import _lib
        torch.cuda.synchronize()
        _lib.poll_kernel_error()


def at(addr: int, nbytes: int, cuda: bool) -> torch.Tensor:
    """The nbytes bytes at a raw address (a device or host-mapped address on the device, a host address on the CPU)
    as a uint8 tensor sharing them."""
    if cuda:
        class _Range:
            __cuda_array_interface__ = dict(shape=(nbytes,), typestr="|u1", data=(addr, False), strides=None, version=3)
        return torch.as_tensor(_Range(), device="cuda")
    import ctypes
    return torch.frombuffer((ctypes.c_uint8 * nbytes).from_address(addr), dtype=torch.uint8)


def _stem_check(what, got, img, bnd, s2d, dtype):
    """got [rows, kpad] of a stem gather of img: every column but "others" bit-exact after one rounding to the map
    type, "others" (channel 4 of the five-channel images, K >= 3) within its bound (exact where that is 0)."""
    kpad = got.shape[-1]
    cin = img.shape[1]
    got = got.double()
    rounded = img.to(dtype).double()
    has_bound = bool(bnd.any())
    if has_bound:
        rounded[:, 4] = img[:, 4]
    ref = R.stem_matrix(rounded, kpad, s2d).to(got.device)
    if not has_bound:
        return exact(what, got, ref)
    b = r16(R.stem_matrix(bnd, kpad, s2d).to(got.device), ref, dtype)
    col = torch.arange(kpad, device=got.device)
    oc = (col < (16 if s2d else 49) * cin) & (col % cin == 4)
    exact(f"{what}: frame / own-mask / pad columns", got[:, ~oc], ref[:, ~oc])
    return bounded(f"{what}: others", got[:, oc], ref[:, oc], b[:, oc])


def _stem_rows(H, W):
    return (H // 2 + 2) * (W // 2 + 2)


@form("stem_gather")
def _():
    def images(A):
        fr, m = A["frame"], A["masks"]
        if m is None:
            return R.stem_images(fr)
        if m.dim() == 5:
            return R.stem_images(fr, m[:, :, 0])
        return R.stem_images(fr, m[:, 0][None])

    def count(A):
        fr, m = A["frame"], A["masks"]
        return fr.shape[0] if m is None else m.shape[0] * m.shape[1] if m.dim() == 5 else m.shape[0]

    def spec(A):
        H, W = A["frame"].shape[-2:]
        N = count(A)
        return {"out": lambda t: [t.reshape(-1, t.shape[-1])[:N * _stem_rows(H, W)]]}

    def check(A, O, fn):
        img, bnd = images(A)
        H, W = A["frame"].shape[-2:]
        got = O["out"].reshape(-1, O["out"].shape[-1])[:count(A) * _stem_rows(H, W)]
        return _stem_check("stem_gather", got, img, bnd, bool(A["s2d"]), O["out"].dtype), {}
    return spec, check


@form("stem_gather_range")
def _():
    def spec(A):
        H, W = A["frame"].shape[-2:]
        return {"out": lambda t: [t.reshape(-1, t.shape[-1])[:A["n"] * _stem_rows(H, W)]]}

    def check(A, O, fn):
        H, W = A["frame"].shape[-2:]
        out = O["out"]
        got = out.reshape(-1, out.shape[-1])[:A["n"] * _stem_rows(H, W)]
        K = A["masks"].shape[0]
        ref = R.stem_reference(A["frame"], A["masks"], A["obj0"], A["n"]).to(got.device)
        exact("stem_gather_range: pad columns", got[:, 80:], torch.zeros_like(got[:, 80:]))
        return bounded("stem_gather_range", got[:, :80], ref, R.stem_tolerance(ref, K, out.dtype == torch.float16)), \
            dict(obj0=int(A["obj0"]), K=K)
    return spec, check


def _first(A, maps):
    return groups_of(_ints(A["first"]), maps)


@form("stem_gather_groups")
def _():
    def spec(A):
        H, W = A["frames"].shape[-2:]
        rows = _stem_rows(H, W)
        gs = _first(A, A["n"])
        return {"out": lambda t: [t.reshape(-1, t.shape[-1])[a * rows:b * rows] for _g, a, b in gs]}

    def check(A, O, fn):
        fr, pl, out = A["frames"], A["planes"], O["out"]
        H, W = fr.shape[-2:]
        rows = _stem_rows(H, W)
        worst = 0.0
        for g, a, b in _first(A, A["n"]):
            img, bnd = R.stem_images(fr[g:g + 1], pl[a + g + 1:b + g + 1, 0][None])
            got = out.reshape(-1, out.shape[-1])[a * rows:b * rows]
            worst = max(worst, _stem_check(f"stem_gather_groups group {g}", got, img, bnd, True, out.dtype))
        return worst, {}
    return spec, check


def _frames_form(name):
    @form(name)
    def _():
        def spec(A):
            n, _c, H, W = A["frames"].shape
            return {"out": lambda t: [t.reshape(-1, t.shape[-1])[:n * _stem_rows(H, W)]]}

        def check(A, O, fn):
            n, _c, H, W = A["frames"].shape
            out = O["out"]
            img, bnd = R.stem_images(A["frames"])
            return _stem_check(name, out.reshape(-1, out.shape[-1])[:n * _stem_rows(H, W)], img, bnd, False,
                               out.dtype), {}
        return spec, check


_frames_form("stem_gather_frames")
_frames_form("stem_gather_frames_tiled")


def _unfold_rows(x, n, h, w, c, ks, stride, dil, pad, ho, wo):
    cols = F.unfold(nchw(interior(x, n, h, w, 0, c)), ks, dilation=dil, padding=pad, stride=stride)
    kk = ks * ks
    assert cols.shape[-1] == ho * wo, "the unfolded map is not the output map"
    cols = cols.reshape(n, c, kk, ho, wo).permute(0, 3, 4, 2, 1).reshape(n, ho, wo, kk * c)
    ref = torch.zeros((n, ho + 2, wo + 2, kk * c), dtype=torch.float64, device=x.device)
    ref[:, 1:-1, 1:-1] = cols
    return ref


@form("gather_s2")
def _():
    def spec(A):
        n, h, w, c, ks = A["n"], A["h"], A["w"], A["c"], A["ks"]
        return {"out": lambda t: [matrix_rows(t, n, h // 2, w // 2, 0, ks * ks * c)]}

    def check(A, O, fn):
        n, h, w, c, ks = A["n"], A["h"], A["w"], A["c"], A["ks"]
        ref = _unfold_rows(A["x"], n, h, w, c, ks, 2, 1, ks // 2, h // 2, w // 2)
        return exact("gather_s2", matrix_rows(O["out"], n, h // 2, w // 2, 0, ks * ks * c), ref), {}
    return spec, check


@form("gather_dilated")
def _():
    def spec(A):
        n, h, w, c = A["n"], A["h"], A["w"], A["c"]
        return {"out": lambda t: [matrix_rows(t, n, h, w, 0, 9 * c)]}

    def check(A, O, fn):
        n, h, w, c, d = A["n"], A["h"], A["w"], A["c"], A["dilation"]
        ref = _unfold_rows(A["x"], n, h, w, c, 3, 1, d, d, h, w)
        return exact(f"gather_dilated d={d}", matrix_rows(O["out"], n, h, w, 0, 9 * c), ref), {}
    return spec, check


@form("maxpool3x3s2")
def _():
    def spec(A):
        n, h, w = A["n"], A["h"], A["w"]
        return {"out": lambda t: [interior(t, n, h // 2, w // 2, 0, t.shape[-1])]}

    def check(A, O, fn):
        n, h, w, x = A["n"], A["h"], A["w"], A["x"]
        ref = F.max_pool2d(nchw(interior(x, n, h, w, 0, x.shape[-1])), 3, 2, 1).permute(0, 2, 3, 1)
        return exact("maxpool3x3s2", interior(O["out"], n, h // 2, w // 2, 0, x.shape[-1]), ref), {}
    return spec, check


def _skip_add_check(what, base, up, h, w, got, dtype):
    """got = base + up2x(up) within 5u (|base| + bilinear |up|) (exact weights, at most 5 roundings per corner
    term), plus one rounding into fp16 maps."""
    u = nchw(up)
    ref = base + R._bilinear(u, h, w)
    bound = r16(5 * R.U * (base.abs() + R._bilinear(u.abs(), h, w)), ref, dtype)
    return bounded(what, nchw(got), ref, bound)


def _relu_bits(what, x, xr):
    if not torch.equal(xr, x.clamp_min(0)):
        raise Mismatch(f"{what}: x_relu != relu(x) at {int((xr != x.clamp_min(0)).sum())} elements")


@form("upsample2x_add")
def _():
    def spec(A):
        n, h, w = A["n"], A["h"], A["w"]
        win = lambda t: [interior(t, n, h, w, 0, t.shape[-1])]  # noqa: E731
        return {"x": win, "x_relu": win}

    def check(A, O, fn):
        n, h, w, x = A["n"], A["h"], A["w"], A["x"]
        C = x.shape[-1]
        if A["skip"] is not None:
            sk = A["skip"]
            base = nchw(interior(sk, sk.shape[0], h, w, 0, C)).repeat_interleave(n // sk.shape[0], 0)
        else:
            base = nchw(interior(x, n, h, w, 0, C))
        got = interior(O["x"], n, h, w, 0, C)
        r = _skip_add_check("upsample2x_add", base, interior(A["up"], n, h // 2, w // 2, 0, C), h, w, got, x.dtype)
        if O.get("x_relu") is not None:
            _relu_bits("upsample2x_add", got, interior(O["x_relu"], n, h, w, 0, C))
        return r, dict(skip_n=0 if A["skip"] is None else A["skip"].shape[0])
    return spec, check


@form("upsample2x_add_groups")
def _():
    def spec(A):
        h, w = A["h"], A["w"]
        gs = _first(A, A["n"])
        win = lambda t: [t[a:b, 1:h + 1, 1:w + 1] for _g, a, b in gs]  # noqa: E731
        return {"x": win, "x_relu": win}

    def check(A, O, fn):
        h, w, sk = A["h"], A["w"], A["skip"]
        C = A["x"].shape[-1]
        worst = 0.0
        for g, a, b in _first(A, A["n"]):
            base = nchw(interior(sk[g:g + 1], 1, h, w, 0, C)).expand(b - a, -1, -1, -1)
            got = O["x"][a:b, 1:h + 1, 1:w + 1]
            worst = max(worst, _skip_add_check(f"upsample2x_add_groups group {g}", base,
                                               A["up"][a:b, 1:h // 2 + 1, 1:w // 2 + 1], h, w, got, A["x"].dtype))
            if O.get("x_relu") is not None:
                _relu_bits(f"upsample2x_add_groups group {g}", got, O["x_relu"][a:b, 1:h + 1, 1:w + 1])
        return worst, {}
    return spec, check


def _copy_ref(src, maps, h, w, coff, c, relu):
    v = interior(src, maps, h, w, coff, c).double()
    return v.clamp_min(0) if relu else v


@form("halo_copy")
def _():
    def spec(A):
        n, h, w, c, d = A["n"], A["h"], A["w"], A["c"], A["dst_coff"]
        return {"dst": lambda t: [interior(t, n, h, w, d, c)]}

    def check(A, O, fn):
        n, h, w, c, src = A["n"], A["h"], A["w"], A["c"], A["src"]
        ref = _copy_ref(src, src.shape[0], h, w, A["src_coff"], c, A["relu"]).repeat_interleave(n // src.shape[0], 0)
        return exact("halo_copy", interior(O["dst"], n, h, w, A["dst_coff"], c), ref), {}
    return spec, check


@form("halo_copy_groups")
def _():
    def spec(A):
        h, w, c, d = A["h"], A["w"], A["c"], A["dst_coff"]
        gs = _first(A, A["n"])
        return {"dst": lambda t: [t[a:b, 1:h + 1, 1:w + 1, d:d + c] for _g, a, b in gs]}

    def check(A, O, fn):
        h, w, c, d, src = A["h"], A["w"], A["c"], A["dst_coff"], A["src"]
        for g, a, b in _first(A, A["n"]):
            ref = _copy_ref(src[g:g + 1], 1, h, w, A["src_coff"], c, A["relu"]).expand(b - a, -1, -1, -1)
            exact(f"halo_copy_groups group {g}", O["dst"][a:b, 1:h + 1, 1:w + 1, d:d + c], ref)
        return 0.0, {}
    return spec, check


@form("halo_to_pixels")
def _():
    def spec(A):
        return {"out": lambda t: [flat(t, A["n"] * A["h"] * A["w"] * A["c"])]}

    def check(A, O, fn):
        n, h, w, c = A["n"], A["h"], A["w"], A["c"]
        ref = interior(A["halo"], n, h, w, A["coff"], c).reshape(-1)
        return exact("halo_to_pixels", flat(O["out"], n * h * w * c), ref), {}
    return spec, check


@form("halo_to_nchw", returns="out")
def _():
    def spec(A):
        return {"out": lambda t: [flat(t, A["n"] * A["c"] * A["h"] * A["w"])]}

    def check(A, O, fn):
        n, h, w, c = A["n"], A["h"], A["w"], A["c"]
        ref = nchw(interior(A["halo"], n, h, w, A["coff"], c)).reshape(-1)
        return exact("halo_to_nchw", flat(O["out"], n * c * h * w), ref), {}
    return spec, check


@form("nchw_to_halo")
def _():
    def spec(A):
        n, c, h, w = A["x"].shape
        return {"halo": lambda t: [interior(t, n, h, w, A["coff"], c)]}

    def check(A, O, fn):
        x = A["x"]
        n, c, h, w = x.shape
        ref = x.double().permute(0, 2, 3, 1)
        return exact("nchw_to_halo", interior(O["halo"], n, h, w, A["coff"], c), ref.clamp_min(0) if A["relu"] else ref), {}
    return spec, check


@form("bank_from_nchw")
def _():
    def spec(A):
        k, _c, t, h, w = A["keys"].shape
        return {"bank_k": lambda b: [b[:k, :t * h * w]], "bank_v": lambda b: [b[:k, :t * h * w]]}

    def check(A, O, fn):
        k, _c, t, h, w = A["keys"].shape
        for name, src, ch in (("bank_k", A["keys"], 128), ("bank_v", A["values"], 512)):
            exact(f"bank_from_nchw {name}", O[name][:k, :t * h * w], src.permute(0, 2, 3, 4, 1).reshape(k, -1, ch))
        return 0.0, {}
    return spec, check


@form("fusion_gather")
def _():
    def spec(A):
        h, w = A["im"].shape[-2:]
        return {"out_halo": lambda t: [t[:1, 1:h + 1, 1:w + 1]]}

    def check(A, O, fn):
        im = A["im"]
        h, w = im.shape[-2:]
        out = O["out_halo"]
        const = torch.tensor([A["nc"], A["nr"]], dtype=torch.float32, device=im.device).view(1, 2, 1, 1).expand(1, 2, h, w)
        planes = torch.cat([im, A["seg1"], A["seg2"], A["attn"], const], 1).double()
        ref = torch.zeros((1, h, w, out.shape[-1]), dtype=torch.float64, device=im.device)
        ref[..., :9] = planes.permute(0, 2, 3, 1)
        return exact("fusion_gather", out[:1, 1:h + 1, 1:w + 1], ref), {}
    return spec, check


@form("halo_sigmoid_to_plane")
def _():
    def spec(A):
        return {"plane": lambda t: [flat(t, A["h"] * A["w"])]}

    def check(A, O, fn):
        h, w = A["h"], A["w"]
        p = torch.sigmoid(A["halo"][0, 1:h + 1, 1:w + 1, A["coff"]].double()).reshape(-1)
        return bounded("halo_sigmoid_to_plane", flat(O["plane"], h * w), p, R.sigmoid_bound(p)), {}
    return spec, check


@form("halo_avgpool_broadcast")
def _():
    def spec(A):
        return {"out": lambda t: [interior(t, A["n"], A["h"], A["w"], A["out_coff"], A["c"])]}

    def check(A, O, fn):
        n, h, w, c = A["n"], A["h"], A["w"], A["c"]
        win = interior(O["out"], n, h, w, A["out_coff"], c)
        if not bool((win == win[:, :1, :1]).all()):
            raise Mismatch("halo_avgpool_broadcast: the mean is not the same at every pixel")
        mu, b = R.avgpool_reference(nchw(interior(A["x"], n, h, w, A["in_coff"], c)))
        return bounded("halo_avgpool_broadcast", win[:, 0, 0], mu, r16(b, mu, O["out"].dtype)), {}
    return spec, check


@form("upsample_bilinear")
def _():
    def spec(A):
        return {"dst": lambda t: [interior(t, A["n"], A["h"], A["w"], A["dst_coff"], A["c"])]}

    def check(A, O, fn):
        n, c = A["n"], A["c"]
        ref, b = R.bilinear_reference(nchw(interior(A["src"], n, A["hs"], A["ws"], A["src_coff"], c)), A["h"], A["w"])
        got = nchw(interior(O["dst"], n, A["h"], A["w"], A["dst_coff"], c))
        return bounded("upsample_bilinear", got, ref, r16(b, ref, O["dst"].dtype)), {}
    return spec, check


@form("halo_upsample_to_plane", returns="out")
def _():
    def spec(A):
        return {"out": lambda t: [flat(t, A["n"] * A["out_h"] * A["out_w"])]}

    def check(A, O, fn):
        n, H, W = A["n"], A["out_h"], A["out_w"]
        ref, b = R.bilinear_reference(nchw(interior(A["halo"], n, A["hs"], A["ws"], A["coff"], 1)), H, W)
        if A["sigmoid"]:
            p = torch.sigmoid(ref)
            ref, b = p, p * (1 - p) * b + R.sigmoid_bound(p)
        out = O["out"]
        return bounded("halo_upsample_to_plane", flat(out, n * H * W), ref.reshape(-1), b.reshape(-1)), \
            dict(sigmoid=bool(A["sigmoid"]), map0=out.storage_offset() // max(1, H * W))
    return spec, check


# ---- aggregation
def _agg_check(what, p, o_got, K, const_bg=False, hard=False, keep_bg=True):
    """o_got [K+1 or K, ...] against aggregate_reference of the fp32 object probabilities p [K, ...]."""
    o, ob, lg = R.aggregate_reference(p.reshape(K, -1), const_bg)
    got = o_got.reshape(o_got.shape[0], -1)
    sel = slice(None) if keep_bg else slice(1, None)
    if hard:
        hl = 1000 * lg
        top2 = hl.topk(2, 0).values
        clear = top2[0] - top2[1] > HARD_GAP
        onehot = F.one_hot(hl.argmax(0), K + 1).t().double()
        tol = K * math.exp(-(HARD_GAP - 1)) + (K + 1) * 2.0 ** -23
        worst = bounded(f"{what} (hard, where the gap exceeds {HARD_GAP:g})", got[:, clear], onehot[sel][:, clear], tol)
    else:
        worst = bounded(what, got, o[sel], ob[sel])
    if keep_bg:
        s = R.sum_and_range_ratio(got, K)
        if s > 1.0:
            raise Mismatch(f"{what}: [bg, objects] leave [0, 1] or do not sum to 1: {s:.3g}x the bound")
    return worst


def _raw_check(what, logits, maps, h4, w4, coff, raw):
    H, W = 4 * h4, 4 * w4
    lg = nchw(interior(logits, maps, h4, w4, coff, 1))
    p, rb = R.upsample4x_raw_reference(lg, H, W)
    return bounded(what, raw.reshape(maps, 1, H, W), p, rb)


def _u4_form(name):
    @form(name, returns="raw_prob")
    def _():
        def sizes(A):
            G, k = A["groups"], A["k"]
            return G, k, 16 * A["h4"] * A["w4"]

        def spec(A):
            G, k, hw = sizes(A)
            return {"raw_out": lambda t: [flat(t, G * k * hw)], "prob_out": lambda t: [flat(t, G * (k + 1) * hw)]}

        def check(A, O, fn):
            G, k, hw = sizes(A)
            raw, prob = O.get("raw_out"), O.get("prob_out")
            if raw is None and prob is not None:  # the kernel's own raw, from a re-run into scratch
                raw = torch.empty((G * k, 1, 4 * A["h4"], 4 * A["w4"]), dtype=torch.float32, device=prob.device)
                again = torch.empty_like(prob)
                fn(A["logits"], k, A["h4"], A["w4"], A["coff"], raw_out=raw, prob_out=again, groups=G)
                _synced(raw)
                exact(f"{name}: prob of the re-run with raw_out", flat(again, G * (k + 1) * hw),
                      flat(prob, G * (k + 1) * hw))
            worst = _raw_check(f"{name} raw", A["logits"], G * k, A["h4"], A["w4"], A["coff"], flat(raw, G * k * hw))
            if prob is not None:
                for g in range(G):
                    worst = max(worst, _agg_check(f"{name} prob group {g}", raw.reshape(-1)[g * k * hw:(g + 1) * k * hw],
                                                  prob.reshape(-1)[g * (k + 1) * hw:(g + 1) * (k + 1) * hw]
                                                  .view(k + 1, hw), k))
            return worst, dict(K=k, G=G, prob=prob is not None)
        return spec, check


_u4_form("upsample4x_sigmoid_aggregate")
_u4_form("upsample4x_sigmoid_aggregate_planes")


@form("upsample4x_sigmoid_aggregate_groups", returns="raw_prob")
def _():
    def gs(A):
        return [(g, a, b) for g, a, b in _first(A, A["n"]) if b - a <= 16]

    def spec(A):
        hw = 16 * A["h4"] * A["w4"]
        return {"raw_out": lambda t: [flat(t, A["n"] * hw)[a * hw:b * hw] for _g, a, b in gs(A)],
                "prob_out": lambda t: [t.reshape(-1)[(a + g) * hw:(b + g + 1) * hw] for g, a, b in gs(A)]}

    def check(A, O, fn):
        n, hw = A["n"], 16 * A["h4"] * A["w4"]
        raw, prob = O.get("raw_out"), O.get("prob_out")
        groups = len(_ints(A["first"])) - 1
        if raw is None:
            raw = torch.empty((n, 1, 4 * A["h4"], 4 * A["w4"]), dtype=torch.float32, device=prob.device)
            again = torch.full_like(prob, math.nan)
            fn(A["logits"], n, A["h4"], A["w4"], A["first"], A["coff"], raw_out=raw, prob_out=again)
            _synced(raw)
            for g, a, b in gs(A):
                exact(f"upsample4x_sigmoid_aggregate_groups: prob of the re-run, group {g}",
                      again.reshape(-1)[(a + g) * hw:(b + g + 1) * hw], prob.reshape(-1)[(a + g) * hw:(b + g + 1) * hw])
        worst = 0.0
        for g, a, b in gs(A):
            r = raw.reshape(-1)[a * hw:b * hw]
            worst = max(worst, _raw_check(f"upsample4x_sigmoid_aggregate_groups raw group {g}", A["logits"][a:b], b - a,
                                          A["h4"], A["w4"], A["coff"], r))
            if prob is not None:
                worst = max(worst, _agg_check(f"upsample4x_sigmoid_aggregate_groups prob group {g}", r,
                                              prob.reshape(-1)[(a + g) * hw:(b + g + 1) * hw].view(b - a + 1, hw), b - a))
        sizes = tuple(b - a for _g, a, b in gs(A))
        return worst, dict(K=n, G=groups, sizes=sizes, prob=prob is not None)
    return spec, check


def _agg_form(name):
    @form(name, returns="out")
    def _():
        def spec(A):
            return {"out": lambda t: [t]}

        def check(A, O, fn):
            p = A["prob"]
            K = p.shape[0]
            return _agg_check(name, p, O["out"], K, A["const_bg"], A["hard"], A["keep_bg"]), dict(K=K)
        return spec, check


_agg_form("aggregate_wbg")
_agg_form("aggregate_wbg_planes")


@form("argmax_unpad")
def _():
    def spec(A):
        return {"masks_padded": lambda t: [t], "masks_out": lambda t: [t]}

    def check(A, O, fn):
        prob, pad, h, w = A["prob"], A["pad"], A["h"], A["w"]
        ref = torch.argmax(prob.cpu(), 0).to(torch.uint8)  # the CPU argmax: the first maximum wins
        exact("argmax_unpad masks_padded", O["masks_padded"], ref)
        if O.get("masks_out") is not None:
            exact("argmax_unpad masks_out", O["masks_out"], ref[:, 0, pad[2]:pad[2] + h, pad[0]:pad[0] + w])
        return 0.0, dict(pad=tuple(pad), K=prob.shape[0] - 1)
    return spec, check


@form("frames_u8_normalize", returns="out")
def _():
    def spec(A):
        return {"out": lambda t: [t]}

    def check(A, O, fn):
        # the kernel's fp32 operations, in the header's order: v = x / 255, then (v - mean) / std, each rounded once
        x = A["frames_hwc"].cpu().permute(0, 3, 1, 2).float() / 255.0
        ref = (x - torch.tensor(NORM_MEAN).view(1, 3, 1, 1)) / torch.tensor(NORM_STD).view(1, 3, 1, 1)
        return exact("frames_u8_normalize", O["out"].cpu(), ref), {}
    return spec, check


@form("pad2d", returns="out")
def _():
    def spec(A):
        return {"out": lambda t: [t]}

    def check(A, O, fn):
        return exact("pad2d", O["out"], F.pad(A["x"].double(), tuple(A["pad"]))), dict(pad=tuple(A["pad"]))
    return spec, check


@form("store_words")
def _():
    def spec(A):
        return {"dst64": lambda t: [t[:len(list(A["vals64"]))]], "dst32": lambda t: [t[:len(list(A["vals32"]))]]}

    def check(A, O, fn):
        exact("store_words dst64", O["dst64"][:len(list(A["vals64"]))], torch.tensor(list(A["vals64"]), dtype=torch.int64))
        if O.get("dst32") is not None:
            exact("store_words dst32", O["dst32"][:len(list(A["vals32"]))],
                  torch.tensor(list(A["vals32"]), dtype=torch.int32))
        return 0.0, {}
    return spec, check


# ---- attention
def _attn_form(name, weights, streamed):
    @form(name, returns="out")
    def _():
        def spec(A):
            return {"out": lambda t: [t]}

        def check(A, O, fn):
            mk, qk, out = A["mk"], A["qk"], O["out"]
            if weights and not streamed:
                W, Wb = R.attention_reference(mk, qk)
                worst = bounded(name, out, W, Wb)
            elif weights:
                worst = 0.0
                for j0, j1, W, Wb in R.weights_streamed_blocks(mk, qk):
                    worst = max(worst, bounded(f"{name} columns {j0}:{j1}", out[:, j0:j1], W, Wb))
            elif not streamed:
                _W, _Wb, ref, b = R.attention_reference(mk, qk, A["h16"], A["w16"], A["pos"], A["neg"])
                worst = bounded(name, out, ref, b)
            else:
                ref, b, _br, _bad = R.map_reference(mk, qk, A["h16"], A["w16"], A["pos"], A["neg"])
                worst = bounded(name, out, ref, b)
            return worst, dict(hw=mk.shape[0])
        return spec, check


_attn_form("attention_map", False, False)
_attn_form("attention_weights", True, False)
_attn_form("attention_map_streamed", False, True)
_attn_form("attention_weights_streamed", True, True)

# ---- graph staging, result delivery, the GUI overlay
@form("copy_segments")
def _():
    def spec(A):
        return {k: (lambda t: []) for k in ("fixed", "dyn", "nbytes")}  # the tables are read, never written

    def pre(A, hosts):
        """Per segment: (index, destination, bytes, the bytes it must hold after the launch, null)."""
        cuda = A["fixed"].is_cuda
        n = A["n"]
        fixed, dyn, nb = (_ints(A[k])[:n] for k in ("fixed", "dyn", "nbytes"))
        segs = []
        for i, (f, d, b) in enumerate(zip(fixed, dyn, nb)):
            if d == 0:  # a null segment copies nothing: a fixed destination keeps its bytes
                if A["dyn_is_src"] and b > 0:
                    segs.append((i, f, b, at(f, b, cuda).clone(), True))
                continue
            src, dst = (d, f) if A["dyn_is_src"] else (f, d)
            segs.append((i, dst, b, at(src, b, cuda).clone() if b > 0 else None, False))
        return dict(cuda=cuda, segs=segs, nulls=sum(1 for d in dyn if d == 0))

    def check(A, O, fn):
        st = A["_pre"]
        for i, dst, b, want, null in st["segs"]:
            if b > 0:
                exact(f"copy_segments segment {i} ({'null, destination must keep its bytes' if null else f'{b} bytes'})",
                      at(dst, b, st["cuda"]), want)
        return 0.0, dict(dyn_is_src=bool(A["dyn_is_src"]), nulls=st["nulls"], segments=A["n"])
    return spec, check, pre


def _host_of(hosts, addr, nbytes):
    """(tensor, byte offset) of the host registration holding [addr, addr + nbytes), or None."""
    for base, t in hosts:
        size = t.numel() * t.element_size()
        if base <= addr and addr + nbytes <= base + size:
            return t, addr - base
    return None


@form("deliver_planes")
def _():
    def spec(A):
        return {"table": lambda t: [], "planes": lambda t: []}  # read, never written

    def pre(A, hosts):
        """The records of the launch and a copy of every host registration: a delivery writes frame ti's planes and
        labels of its own volume, a null record nothing."""
        nh, nw = A["nh"], A["nw"]
        plane = nh * nw
        words = _ints(A["table"])
        recs, wins = [], {}
        for c in range(A["clips"]):
            r = words[c * 8:(c + 1) * 8]
            k1 = r[4] >> 32
            if r[0] == 0 or not 1 <= k1 <= 256:
                recs.append(None)
                continue
            h, w = r[6] & 0xFFFFFFFF, r[6] >> 32
            spans = [(r[0] + j * r[1] * 4, plane * 4) for j in range(k1)] + [(r[2], plane), (r[3], h * w)]
            where = []
            for a, n in spans:
                hit = _host_of(hosts, a, n)
                if hit is None:
                    raise Mismatch(f"deliver_planes record {c}: address {a:#x} lies in no host registration made while "
                                   "recording")
                wins.setdefault(id(hit[0]), []).append((hit[1], n))
                where.append(hit)
            recs.append(dict(c=c, first=r[4] & 0xFFFFFFFF, k1=k1, pad_l=r[5] & 0xFFFFFFFF, pad_t=r[5] >> 32, h=h, w=w,
                             where=where))
        blocks = [(t, storage_bytes(t).clone(), wins.get(id(t), [])) for _a, t in hosts]
        return dict(recs=recs, blocks=blocks)

    def check(A, O, fn):
        st = A["_pre"]
        nh, nw = A["nh"], A["nw"]
        plane = nh * nw
        for t, before, spans in st["blocks"]:
            changed_outside(before, t, lambda x, spans=spans: [x.reshape(-1).view(torch.uint8)[o:o + n] for o, n in spans],
                            "deliver_planes: host volume (frames other than ti, other volumes, null records)")
        planes = A["planes"].reshape(-1, plane).cpu()
        for r in st["recs"]:
            if r is None:
                continue
            src = planes[r["first"]:r["first"] + r["k1"]]
            byte = lambda i, n: r["where"][i][0].reshape(-1).view(torch.uint8)[r["where"][i][1]:r["where"][i][1] + n]  # noqa: E731
            for j in range(r["k1"]):
                exact(f"deliver_planes record {r['c']} plane {j}", byte(j, plane * 4).view(torch.float32).cpu(), src[j])
            lab = torch.argmax(src, 0).to(torch.uint8)  # the CPU argmax: the first maximum wins
            exact(f"deliver_planes record {r['c']} padded labels", byte(r["k1"], plane).cpu(), lab)
            crop = lab.view(nh, nw)[r["pad_t"]:r["pad_t"] + r["h"], r["pad_l"]:r["pad_l"] + r["w"]].reshape(-1)
            exact(f"deliver_planes record {r['c']} labels", byte(r["k1"] + 1, r["h"] * r["w"]).cpu(), crop)
        return 0.0, dict(nulls=sum(1 for r in st["recs"] if r is None), hosts=sum(1 for r in st["recs"] if r))
    return spec, check, pre


@form("overlay_davis", returns="out")
def _():
    def spec(A):
        return {"out": lambda t: [t]}

    def check(A, O, fn):
        """The kernel's double operations: fl(fl(px alpha) + fl((1 - alpha) colour)) truncated on objects, black on
        their 4-neighbour contour, fl(px 0.6) truncated elsewhere with fade."""
        img, m = A["image"].cpu().double(), A["mask"].cpu().long()
        if m.dim() == 2:
            img, m = img[None], m[None]
        tab = torch.tensor(A["colors"], dtype=torch.uint8).reshape(-1, 3).double()
        alpha = float(A["alpha"])
        col = tab[torch.where(m < tab.shape[0], m, 0)]
        blend = (img * alpha + (1.0 - alpha) * col).trunc()
        obj = m > 0
        nb = torch.zeros_like(obj)
        nb[:, 1:] |= obj[:, :-1]
        nb[:, :-1] |= obj[:, 1:]
        nb[:, :, 1:] |= obj[:, :, :-1]
        nb[:, :, :-1] |= obj[:, :, 1:]
        rest = (img * 0.6).trunc() if A["fade"] else img
        ref = torch.where(obj[..., None], blend, torch.where(nb[..., None], torch.zeros_like(img), rest))
        return exact("overlay_davis", O["out"].cpu().reshape(ref.shape), ref), dict(fade=bool(A["fade"]))
    return spec, check



# ------------------------------------------------------------------ one launch
def _tensors(A):
    return {k: v for k, v in A.items() if torch.is_tensor(v)}


def _desc(k, v):
    if torch.is_tensor(v):
        d = (tuple(v.shape), str(v.dtype), v.untyped_storage().nbytes(), v.storage_offset())
        if k in ("first", "nbytes"):
            return d + (tuple(_ints(v)),)
        if k == "dyn":  # the null segments, not the addresses of the frame
            return d + (tuple(x == 0 for x in _ints(v)),)
        if k == "table":  # the null records
            return d + (tuple(x == 0 for x in _ints(v)[::8]),)
        return d
    if isinstance(v, (list, tuple)) and k != "pad":
        return ("seq", len(v))
    return v


def signature(name, A) -> tuple:
    return (name,) + tuple((k, _desc(k, v)) for k, v in A.items())


def _returned(f: Form, A: dict, res) -> dict:
    """The outputs the launch allocated and returned."""
    if f.returns == "out":
        return {"out": res}
    if f.returns == "raw_prob":
        raw, prob = res
        return {"raw_out": raw, "prob_out": prob}
    return {}


def checked(name: str, fn, args=(), kw=None, *, max_bytes: int = SNAPSHOT_BYTES, on_launch=None, hosts=()):
    """Snapshot, run and check one launch of form `name` through fn (the real operator, or an emulation on the CPU).
    `hosts`: the (address, tensor) of every host registration (ops.host_register) a delivery may write through.
    Returns (the launch's result, the record of the table); the record is None when an output allocation is above
    max_bytes (counted, not checked)."""
    f = FORMS[name]
    A = bind(fn, args, kw or {})
    wins = f.spec(A)
    outs = {k: A[k] for k in wins if A.get(k) is not None}
    if any(t.untyped_storage().nbytes() > max_bytes for t in outs.values()):
        return fn(*args, **(kw or {})), None
    before = {k: storage_bytes(t).clone() for k, t in outs.items()}
    A0 = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in A.items()}
    if f.pre is not None:
        A0["_pre"] = f.pre(A, hosts)
    res = fn(*args, **(kw or {}))
    if on_launch is not None:
        on_launch()
    O = dict(outs)
    for k, t in _returned(f, A, res).items():
        if t is not None and O.get(k) is None:
            O[k] = t
    for k, t in outs.items():
        changed_outside(before[k], t, wins[k], f"{name}: {k}")
    for k, t in O.items():
        if t.is_floating_point():
            for v in wins[k](t):
                if not bool(torch.isfinite(v).all()):
                    raise Mismatch(f"{name}: {k} not finite in its window")
    worst, facts = f.check(A0, O, fn)
    rec = dict(form=name, ratio=worst, **facts)
    rec["dtypes"] = tuple(sorted({_sym(t) for t in _tensors(A).values() if t.is_floating_point()}))
    maps = [t for t in O.values() if t is not None and t.is_floating_point()]
    rec["act"] = _sym(maps[0]) if maps else None  # the type of the maps the launch writes
    firsts = _ints(A["first"]) if torch.is_tensor(A.get("first")) else None
    if firsts is not None:
        maps = A.get("n")
        rec["group_sizes"] = tuple(b - a for _g, a, b in groups_of(firsts, maps))
    rec["prefix"] = any(_maps(A, t) < _alloc_maps(t) for t in outs.values() if t.dim() >= 2)
    return res, rec


def _alloc_maps(t) -> int:
    """Maps (leading-dimension entries) of t's shape that its whole allocation holds."""
    return t.untyped_storage().nbytes() // max(1, t[0].numel() * t.element_size())


def _maps(A, t) -> int:
    """Maps of t that the launch takes part with: its `n` where it has one, else the view's leading dimension."""
    n = A.get("n")
    return min(n, t.shape[0]) if isinstance(n, int) and t.dim() == 4 else t.shape[0]


# ------------------------------------------------------------------ the recorder
class OpCensus:
    """Recorder of operator launches; `record(s)` checks every eager launch of scenario s."""

    def __init__(self, max_bytes: int = SNAPSHOT_BYTES):
        self.max_bytes = max_bytes
        self.records = []
        self.seen = Counter()
        self.checked = Counter()
        self.captured = Counter()
        self.too_big = Counter()
        self.hosts = []  # (address, tensor) of the host registrations made while recording
        self._sigs = set()

    @contextlib.contextmanager
    def record(self, scenario: str):
        from mivos_b200 import ops
        saved = {name: getattr(ops, name) for name in tuple(FORMS) + ("host_register",)}
        for name in FORMS:
            setattr(ops, name, self._wrap(scenario, name, saved[name]))
        register = saved["host_register"]

        def host_register(t):
            addr = register(t)
            self.hosts.append((addr, t))
            return addr
        ops.host_register = host_register
        try:
            yield self
        finally:
            for name, fn in saved.items():
                setattr(ops, name, fn)

    def _wrap(self, scenario, name, fn):
        def launch(*args, **kw):
            return self._launch(scenario, name, fn, args, kw)
        launch.__signature__ = inspect.signature(fn)
        return launch

    def _launch(self, scenario, name, fn, args, kw):
        A = bind(fn, args, kw)
        ts = list(_tensors(A).values())
        cuda = bool(ts) and ts[0].is_cuda
        if cuda and torch.cuda.is_current_stream_capturing():
            self.captured[scenario] += 1
            return fn(*args, **kw)
        self.seen[scenario] += 1
        if cuda:
            torch.cuda.synchronize()
        sig = signature(name, A)
        if sig in self._sigs:
            return fn(*args, **kw)
        self._sigs.add(sig)

        def sync():
            if cuda:
                from mivos_b200 import _lib
                torch.cuda.synchronize()
                _lib.poll_kernel_error()
        res, rec = checked(name, fn, args, kw, max_bytes=self.max_bytes, on_launch=sync, hosts=self.hosts)
        if rec is None:
            self.too_big[scenario] += 1
        else:
            self.records.append(dict(rec, scenario=scenario))
            self.checked[scenario] += 1
        return res

    def table(self) -> str:
        lines = [f"{'form':38s} {'launches':>8s} {'types':12s} {'worst err/bound':>15s}  scenarios"]
        by = {}
        for r in self.records:
            by.setdefault(r["form"], []).append(r)
        for name in sorted(by):
            rs = by[name]
            types = ",".join(sorted({d for r in rs for d in r["dtypes"]}))
            sc = sorted({r["scenario"] for r in rs})
            lines.append(f"{name:38s} {len(rs):8d} {types:12s} {max(r['ratio'] for r in rs):15.3g}  "
                         f"{', '.join(sc[:4])}{' ...' if len(sc) > 4 else ''}")
        return "\n".join(lines)

    def summary(self) -> str:
        out = []
        for s in self.seen:
            rs = [r for r in self.records if r["scenario"] == s]
            out.append(f"{s}: {self.seen[s]} operator launches seen, {self.checked[s]} checked ({len({r['form'] for r in rs})} "
                       f"forms), {self.too_big[s]} above the snapshot limit, worst err/bound "
                       f"{max((r['ratio'] for r in rs), default=0.0):.3g}")
        return "\n".join(out)
