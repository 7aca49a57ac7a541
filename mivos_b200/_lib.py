"""ctypes binding of the C ABI declared in include/mivos_b200.h.

The shared library is built in-tree by ``__graft_entry__.build()`` / ``make -C mivos_b200/csrc``.
There is no fallback: if the library is missing, or the device is not sm_90, every op raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmivos_b200.so")


class MivosError(RuntimeError):
    pass


class ConvArgs(C.Structure):
    """Mirror of ``mivos_conv_args`` (include/mivos_b200.h)."""

    _fields_ = [
        ("in_", C.c_void_p),
        ("in_rows", C.c_int64),
        ("in_cstride", C.c_int),
        ("in_coff", C.c_int),
        ("n", C.c_int),
        ("h", C.c_int),
        ("w", C.c_int),
        ("cin_pad", C.c_int),
        ("taps", C.c_int),
        ("weight", C.c_void_p),
        ("bias", C.c_void_p),
        ("cout", C.c_int),
        ("cout_pad", C.c_int),
        ("out", C.c_void_p),
        ("out_cstride", C.c_int),
        ("out_coff", C.c_int),
        ("residual", C.c_void_p),
        ("res_cstride", C.c_int),
        ("res_coff", C.c_int),
        ("out_relu", C.c_void_p),
        ("out_relu_cstride", C.c_int),
        ("out_relu_coff", C.c_int),
        ("relu", C.c_int),
        ("in_f16", C.c_int),
        ("out_f16", C.c_int),
        ("splitk_ws", C.c_void_p),
        ("splitk_ws_bytes", C.c_int64),
    ]


_p = C.c_void_p
_i = C.c_int
_l = C.c_int64
_f = C.c_float

# name -> (restype, argtypes); the test-suite checks every symbol in the header is listed here
# and exported by the library.
SIGNATURES = {
    "mivos_abi_version": (_i, []),
    "mivos_last_error": (C.c_char_p, []),
    "mivos_check_device": (_i, []),
    "mivos_poll_kernel_error": (_i, [_p, C.POINTER(_i)]),
    "mivos_launch_count": (_l, []),
    "mivos_add_launch_count": (_l, [_l]),
    "mivos_store_i32": (_i, [_p, _i, _i, _i, _i, _i, _p]),
    "mivos_store_words": (_i, [_p, _i, _p, _p, _i, _i, _i, _i, _i, _p]),
    "mivos_copy_segments": (_i, [_p, _p, _p, _i, _i, _l, _p]),
    "mivos_deliver_planes": (_i, [_p, _p, _i, _i, _i, _p]),
    "mivos_host_register": (_i, [_p, _l, C.POINTER(_p)]),
    "mivos_host_unregister": (_i, [_p]),
    "mivos_conv_gemm": (_i, [C.POINTER(ConvArgs), _p]),
    "mivos_conv_tile_override": (_i, [_i, _i]),
    "mivos_conv_plan": (_i, [C.POINTER(ConvArgs), _i, C.POINTER(_i), C.POINTER(_i)]),
    "mivos_conv_plan_residency": (_i, [C.POINTER(ConvArgs), _i, C.POINTER(_i)]),
    "mivos_conv_residency_override": (_i, [_i]),
    "mivos_stem_gather": (_i, [_p, _p, _i, _i, _i, _p, _i, _i, _i, _l, _l, _p]),
    "mivos_stem_gather_s2d": (_i, [_p, _p, _i, _i, _i, _p, _i, _i, _i, _l, _l, _p]),
    "mivos_stem_gather_s2d_range": (_i, [_p, _p, _i, _i, _i, _i, _i, _p, _i, _i, _p]),
    "mivos_gather_s2": (_i, [_p, _i, _i, _i, _i, _i, _i, _p, _i, _i, _p]),
    "mivos_maxpool3x3s2": (_i, [_p, _i, _i, _i, _i, _p, _i, _p]),
    "mivos_upsample2x_add": (_i, [_p, _p, _i, _i, _i, _i, _p, _p, _i, _i, _p]),
    "mivos_halo_copy": (_i, [_p, _i, _i, _i, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "mivos_halo_to_nchw": (_i, [_p, _i, _i, _i, _i, _i, _i, _p, _i, _p]),
    "mivos_nchw_to_halo": (_i, [_p, _i, _i, _i, _i, _p, _i, _i, _i, _i, _p]),
    "mivos_halo_to_pixels": (_i, [_p, _i, _i, _i, _i, _i, _i, _p, _p]),
    "mivos_bank_write": (_i, [_p, _i, _i, _i, _i, _i, _i, _p, _p, _l, _i, _p, _p]),
    "mivos_bank_write_sets": (_i, [_p, _i, _i, _i, _i, _i, _i, _i, _p, _p, _l, _i, _p, _p]),
    "mivos_bank_from_nchw": (_i, [_p, _p, _i, _i, _i, _p, _p, _l, _p]),
    "mivos_memory_read_workspace": (_l, [_i, _l, _i, _i]),
    "mivos_memory_read": (_i, [_p, _p, _l, _i, _l, _p, _i, _i, _i, _p, _i, _i, _i, _i, _p, _p, _p, _l, _i, _p, _i, _p]),
    "mivos_memory_read_sets": (_i, [_p, _p, _l, _i, _l, _p, _i, _i, _i, _p, _i, _i, _i, _i, _p, _p, _p, _l, _i, _p, _i, _p]),
    "mivos_memory_read_dense_sets": (_i, [_p, _p, _l, _i, _l, _p, _i, _i, _p, _i, _i, _i, _i, _p, _l, _p, _i, _p]),
    "mivos_memory_read_wide_sets": (_i, [_p, _p, _l, _i, _l, _p, _i, _i, _i, _p, _i, _i, _i, _i, _p, _p, _p, _l, _p, _i, _p]),
    "mivos_memory_read_groups": (_i, [_p, _p, _l, _i, _l, _p, _i, _i, _p, _i, _p, _i, _i, _i, _i, _p, _p, _p, _l, _i, _p, _i, _p]),
    "mivos_memory_read_dense_groups": (_i, [_p, _p, _l, _i, _l, _p, _i, _i, _p, _p, _i, _i, _i, _i, _p, _l, _p, _i, _p]),
    "mivos_memory_read_wide_groups": (_i, [_p, _p, _l, _i, _l, _p, _i, _i, _p, _i, _p, _i, _i, _i, _i, _p, _p, _p, _l, _p, _i, _p]),
    "mivos_bank_write_groups": (_i, [_p, _i, _i, _p, _i, _i, _i, _i, _i, _p, _p, _l, _i, _p, _p]),
    "mivos_stem_gather_s2d_groups": (_i, [_p, _p, _i, _i, _p, _i, _i, _p, _i, _i, _l, _p]),
    "mivos_upsample2x_add_groups": (_i, [_p, _p, _i, _i, _i, _i, _p, _p, _i, _p, _i, _p]),
    "mivos_halo_copy_groups": (_i, [_p, _i, _p, _i, _i, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "mivos_upsample4x_sigmoid_aggregate_groups": (_i, [_p, _i, _i, _p, _i, _i, _i, _i, _p, _p, _p]),
    "mivos_memory_read_stats": (_i, [_p, _i, _l, _i, _i, C.POINTER(_l)]),
    "mivos_memory_read_dense_workspace": (_l, [_i, _l, _i]),
    "mivos_memory_read_dense": (_i, [_p, _p, _l, _i, _l, _p, _i, _i, _p, _i, _i, _i, _i, _p, _l, _p, _i, _p]),
    "mivos_memory_read_wide_workspace": (_l, [_i, _l, _i, _i]),
    "mivos_memory_read_wide": (_i, [_p, _p, _l, _i, _l, _p, _i, _i, _i, _p, _i, _i, _i, _i, _p, _p, _p, _l, _p, _i, _p]),
    "mivos_upsample4x_sigmoid_aggregate": (_i, [_p, _i, _i, _i, _i, _i, _p, _p, _i, _p]),
    "mivos_aggregate_wbg": (_i, [_p, _i, _l, _i, _i, _p, _p]),
    "mivos_upsample4x_sigmoid_aggregate_planes": (_i, [_p, _i, _i, _i, _i, _i, _p, _p, _i, _p]),
    "mivos_aggregate_wbg_planes": (_i, [_p, _i, _l, _i, _i, _p, _p]),
    "mivos_argmax_unpad": (_i, [_p, _i, _i, _i, _i, _i, _i, _i, _i, _p, _p, _p]),
    "mivos_frames_u8_normalize": (_i, [_p, _i, _i, _i, _p, _p]),
    "mivos_pad2d": (_i, [_p, _i, _i, _i, _i, _i, _i, _i, _p, _p]),
    "mivos_attention_map": (_i, [_p, _p, _i, _i, _p, _p, _p, _p, _p]),
    "mivos_attention_weights": (_i, [_p, _p, _i, _p, _p, _p]),
    "mivos_attention_plan": (_i, [_i, C.POINTER(_i)]),
    "mivos_attention_map_streamed": (_i, [_p, _p, _i, _i, _p, _p, _p, _p, _p]),
    "mivos_attention_weights_streamed": (_i, [_p, _p, _i, _p, _p, _p]),
    "mivos_fusion_gather": (_i, [_p, _p, _p, _p, _f, _f, _i, _i, _p, _i, _i, _p]),
    "mivos_halo_sigmoid_to_plane": (_i, [_p, _i, _i, _i, _i, _p, _p]),
    "mivos_stem_gather_frames": (_i, [_p, _i, _i, _i, _i, _p, _i, _i, _p]),
    "mivos_stem_frames_plan": (_i, [_i, _i, _i, C.POINTER(_i)]),
    "mivos_stem_gather_frames_tiled": (_i, [_p, _i, _i, _i, _p, _i, _i, _p]),
    "mivos_gather_dilated": (_i, [_p, _i, _i, _i, _i, _i, _i, _p, _i, _i, _p]),
    "mivos_halo_avgpool_broadcast": (_i, [_p, _i, _i, _i, _i, _i, _i, _p, _i, _i, _i, _p]),
    "mivos_upsample_bilinear": (_i, [_p, _i, _i, _i, _i, _i, _p, _i, _i, _i, _i, _i, _i, _p]),
    "mivos_halo_upsample_to_plane": (_i, [_p, _i, _i, _i, _i, _i, _i, _i, _i, _p, _p]),
    "mivos_overlay_davis": (_i, [_p, _p, _i, _i, _i, _p, _i, C.c_double, _i, _p, _p]),
}

_lib = None


ABI_VERSION = 4  # include/mivos_b200.h: MIVOS_ABI_VERSION


def load() -> C.CDLL:
    """Load the shared library (no device needed) and bind every declared symbol."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MivosError(
            f"{LIB_PATH} not built. Run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C mivos_b200/csrc`). There is no CPU or PyTorch fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if a symbol is missing: fail loudly
        fn.restype = res
        fn.argtypes = args
    got = lib.mivos_abi_version()
    if got != ABI_VERSION:
        raise MivosError(f"{LIB_PATH} has ABI version {got}, this package binds version {ABI_VERSION}: rebuild it "
                         "(python -c 'import __graft_entry__ as g; g.build()')")
    _lib = lib
    return lib


_device_ok = False


def lib() -> C.CDLL:
    """Library handle for launching work: also verifies the current device is sm_90."""
    global _device_ok
    l = load()
    if not _device_ok:
        rc = l.mivos_check_device()
        if rc != 0:
            raise MivosError(f"mivos_check_device failed ({rc}): {l.mivos_last_error().decode()}")
        _device_ok = True
    return l


def require_cuda_device(device, who: str) -> None:
    """The one place the host classes insist on a CUDA device: there is no CPU path.  (tests/abi_emulator.py
    replaces this guard — and every operator — to exercise the host logic alone on the CPU.)"""
    import torch
    if torch.device(device).type != "cuda":
        raise MivosError(f"{who} must be on a CUDA device (.cuda() / .to('cuda:0')); got {device!r}: mivos_b200 has no CPU path")


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().mivos_last_error().decode(errors="replace")
        raise MivosError(f"{what or 'mivos call'} failed with code {rc}: {msg}")


def poll_kernel_error(stream_ptr: int = 0) -> None:
    code = C.c_int(0)
    rc = lib().mivos_poll_kernel_error(C.c_void_p(stream_ptr), C.byref(code))
    check(rc, f"kernel error flag (code {code.value})")
