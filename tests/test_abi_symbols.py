"""CPU: the C-ABI library loads without a GPU and exports every symbol the header declares, and
the ctypes table binds exactly that set (no compute calls here)."""
import os
import re

from mivos_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "mivos_b200.h")).read()
    return set(re.findall(r"MIVOS_API\s+[\w\s\*]+?\b(mivos_\w+)\s*\(", src))


def test_header_symbols_are_bound_and_exported():
    decl = _declared()
    assert len(decl) >= 25
    assert decl == set(_lib.SIGNATURES), (decl ^ set(_lib.SIGNATURES))
    lib = _lib.load()
    for name in decl:
        assert hasattr(lib, name), name
    assert lib.mivos_abi_version() == _lib.ABI_VERSION == 4  # include/mivos_b200.h: MIVOS_ABI_VERSION


def test_no_torch_types_in_signatures():
    src = open(os.path.join(ROOT, "include", "mivos_b200.h")).read()
    code = re.sub(r"/\*.*?\*/", "", src, flags=re.S)  # declarations only, comments stripped
    assert "torch" not in code.lower() and "at::" not in code and "Tensor" not in code and "std::" not in code


def test_workspace_query_runs_without_gpu():
    lib = _lib.load()
    n = lib.mivos_memory_read_workspace(1, 20 * 1620, 1620, 20)
    assert n > 0
    assert lib.mivos_memory_read_workspace(1, 100, 100, 65) == -1  # top_k above the supported 64


def test_product_path_never_imports_the_oracle():
    imp = re.compile(r"^\s*(from\s+oracle|import\s+oracle|from\s+\.\.?oracle|import\s+abi_emulator|from\s+abi_emulator)", re.M)
    pkg = os.path.join(ROOT, "mivos_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            assert not imp.search(open(os.path.join(pkg, fn)).read()), fn
    for fn in ("inference_core.py", "model/propagation/prop_net.py", "model/fusion_net.py", "model/aggregate.py", "util/tensor_util.py",
               "model/s2m/s2m_network.py", "interact/s2m_controller.py"):
        assert not imp.search(open(os.path.join(ROOT, fn)).read())
    for fn in os.listdir(os.path.join(pkg, "csrc")):
        if fn.endswith((".cu", ".cuh", ".h")):
            assert "oracle" not in open(os.path.join(pkg, "csrc", fn)).read(), fn


def test_argument_validation_fails_loudly_without_touching_a_device():
    """Every entry point validates its arguments before any CUDA call and reports through the return
    code + mivos_last_error() (include/mivos_b200.h: MIVOS_ERR_INVALID = -1); no exception crosses the ABI."""
    import ctypes as C
    lib = _lib.load()
    null, one = C.c_void_p(0), C.c_void_p(16)
    assert lib.mivos_gather_dilated(null, 1, 4, 4, 32, 32, 2, null, 288, 1, null) == -1
    assert b"gather_dilated" in lib.mivos_last_error()
    assert lib.mivos_gather_dilated(one, 1, 4, 4, 30, 32, 2, one, 288, 1, null) == -1  # c not a multiple of the vector width
    assert lib.mivos_stem_gather_frames(one, 1, 4, 32, 32, one, 320, 1, null) == -1  # 4 input channels
    assert b"3 or 6" in lib.mivos_last_error()
    # the first frame width each stem gather refuses for want of shared memory (227 KB per CTA); the width 2 below is
    # the widest admitted, tests/test_gpu_ops_ragged.py runs it for the 6-channel fp32 form
    for w, cin, f16 in ((2762, 3, 0), (5530, 3, 1), (1656, 5, 0), (3316, 5, 1)):
        masks = one if cin == 5 else null
        assert lib.mivos_stem_gather(one, masks, 1, 2, w, one, 256, f16, 1, 0, 0, null) == -1, (w, cin, f16)
        assert b"shared memory" in lib.mivos_last_error()
    for w, cin, f16 in ((9678, 3, 0), (19364, 3, 1), (5804, 5, 0), (11616, 5, 1)):
        masks = one if cin == 5 else null
        assert lib.mivos_stem_gather_s2d(one, masks, 1, 2, w, one, 96, f16, 1, 0, 0, null) == -1, (w, cin, f16)
        assert b"shared memory" in lib.mivos_last_error()
    for w, f16 in ((1378, 0), (2762, 1)):
        assert lib.mivos_stem_gather_frames(one, 1, 6, 2, w, one, 320, f16, null) == -1, (w, f16)
        assert b"shared memory" in lib.mivos_last_error()
    assert lib.mivos_halo_avgpool_broadcast(one, 1, 4, 4, 64, 64, 8, one, 64, 0, 1, null) == -1  # window beyond the stride
    assert lib.mivos_upsample_bilinear(one, 1, 0, 4, 32, 0, one, 8, 8, 32, 0, 32, 0, null) == -1
    assert lib.mivos_halo_upsample_to_plane(one, 1, 4, 4, 32, 32, 16, 16, 0, one, null) == -1  # coff == cstride
    assert lib.mivos_overlay_davis(one, one, 1, 4, 4, one, 7, C.c_double(1.5), 0, one, null) == -1
    assert b"alpha" in lib.mivos_last_error()
    assert lib.mivos_overlay_davis(one, one, 1, 4, 4, one, 0, C.c_double(0.5), 0, one, null) == -1
    assert lib.mivos_attention_map(one, one, -1, -1, one, one, one, one, null) == -1  # negative grid, positive product
    assert b"attention_map" in lib.mivos_last_error()
    assert lib.mivos_attention_map(one, one, 64, 109, one, one, one, one, null) == -1  # 6976 keys: above the 220 KB tile
    assert b"attention_map" in lib.mivos_last_error()
    assert lib.mivos_attention_weights(one, one, 6976, one, one, null) == -1
    assert b"attention_weights" in lib.mivos_last_error()
    a = _lib.ConvArgs()
    assert lib.mivos_conv_gemm(C.byref(a), null) == -1 and b"conv_gemm" in lib.mivos_last_error()
    with __import__("pytest").raises(_lib.MivosError):
        _lib.check(-1, "probe")


def test_every_ctypes_call_site_passes_the_declared_number_of_arguments():
    """The CPU suite drives the host code over the emulated operators, so a wrapper in mivos_b200/ops.py that calls its
    C entry point with the wrong number of arguments would only surface on the GPU box: count them here."""
    src = open(os.path.join(ROOT, "mivos_b200", "ops.py")).read()
    seen = 0
    for name, (_, args) in _lib.SIGNATURES.items():
        for m in re.finditer(r"\b" + name + r"\(", src):
            i, depth, commas, any_arg = m.end(), 1, 0, False
            while depth > 0:
                ch = src[i]
                if ch in "([{":
                    depth += 1
                elif ch in ")]}":
                    depth -= 1
                elif ch == "," and depth == 1:
                    commas += 1
                elif not ch.isspace():
                    any_arg = True
                i += 1
            assert (commas + 1 if any_arg else 0) == len(args), f"{name}: call passes {commas + 1} arguments, signature has {len(args)}"
            seen += 1
    assert seen >= 25
