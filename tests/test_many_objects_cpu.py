"""CPU: clips of 17 to 255 objects without a device — the object-chunk plan, the object-count limit, argument
rejection by the new entry points before any CUDA call, the goldens of oracle/gen_golden_objects.py against the
oracle, and that the GPU tests' bounds catch the two mistakes an object-chunked path could make (an "others" channel
summed over the chunk only, a softmax without the background)."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from mivos_b200 import _lib, ops
from mivos_b200.engine import CHUNK_OBJECTS, object_chunks
from oracle import gen_golden_objects as GO
from oracle import stm_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24


def test_object_chunk_plan():
    assert object_chunks(1) == [(0, 1)] and object_chunks(16) == [(0, 16)]
    assert object_chunks(17) == [(0, 9), (9, 8)]
    assert object_chunks(255) == [(i * 16, 16) for i in range(15)] + [(240, 15)]
    for K in range(1, 256):
        ch = object_chunks(K)
        sizes = [n for _, n in ch]
        assert len(ch) == -(-K // CHUNK_OBJECTS) and sum(sizes) == K
        assert max(sizes) <= CHUNK_OBJECTS and max(sizes) - min(sizes) <= 1 and sizes == sorted(sizes, reverse=True)
        assert [k0 for k0, _ in ch] == [sum(sizes[:i]) for i in range(len(ch))]


def test_object_count_limit():
    for k in (1, 17, 255):
        ops.check_objects(k, "x")
    for k in (0, 256, -1):
        with pytest.raises(_lib.MivosError, match="1 to 255"):
            ops.check_objects(k, "InferenceCore")
        with pytest.raises(_lib.MivosError, match="1 to 255"):
            ops.aggregate_any(torch.zeros(max(k, 0), 1, 2, 2))


def test_new_entry_points_validate_without_a_device():
    lib = _lib.load()
    null, p = C.c_void_p(0), C.c_void_p(256)
    before = lib.mivos_launch_count()
    assert lib.mivos_aggregate_wbg_planes(p, 256, 16, 1, 0, p, null) == -1
    assert b"256 objects" in lib.mivos_last_error()
    assert lib.mivos_aggregate_wbg_planes(p, 0, 16, 1, 0, p, null) == -1
    assert lib.mivos_aggregate_wbg_planes(null, 17, 16, 1, 0, p, null) == -1
    assert lib.mivos_aggregate_wbg_planes(p, 17, 0, 1, 0, p, null) == -1
    assert lib.mivos_upsample4x_sigmoid_aggregate_planes(p, 256, 2, 2, 32, 0, null, p, 1, null) == -1
    assert lib.mivos_upsample4x_sigmoid_aggregate_planes(p, 17, 2, 2, 32, 32, null, p, 1, null) == -1
    assert lib.mivos_upsample4x_sigmoid_aggregate_planes(p, 17, 2, 2, 32, 0, null, null, 1, null) == -1
    assert lib.mivos_upsample4x_sigmoid_aggregate_planes(p, 17, 2, 2, 32, 0, null, p, 0, null) == -1
    for obj0, n in ((-1, 2), (0, 0), (16, 2)):
        assert lib.mivos_stem_gather_s2d_range(p, p, 17, obj0, n, 32, 32, p, 96, 0, null) == -1
        assert b"stem_gather_s2d_range" in lib.mivos_last_error()
    assert lib.mivos_stem_gather_s2d_range(p, null, 17, 0, 2, 32, 32, p, 96, 0, null) == -1
    assert lib.mivos_stem_gather_s2d_range(p, p, 17, 0, 2, 31, 32, p, 96, 0, null) == -1
    assert lib.mivos_launch_count() == before


def test_goldens_match_the_oracle(golden):
    """The reference's outputs equal the oracle's (MANIFEST: 0.0 and equal masks), and the aggregation goldens are
    reproduced by the oracle from their seeds."""
    man = json.load(open(os.path.join(ROOT, "tests", "golden", "MANIFEST_objects.json")))
    for key, v in man.items():
        if key.endswith("_oracle_vs_reference"):
            assert v == 0.0, key
        if key.endswith("_masks_equal"):
            assert all(v), key
    g = golden("objects.npz")
    for K in GO.AGG_K:
        p = GO.agg_inputs(K)
        assert np.array_equal(O.aggregate_wbg(p, keep_bg=True, hard=True).numpy(), g[f"agg_K{K}_wbg_hard"])
        assert np.array_equal(O.aggregate_wbg(p, keep_bg=True).numpy(), g[f"agg_K{K}_wbg_soft"])
    for K in GO.CLIPS:
        T = GO.CLIPS[K][0]
        assert g[f"clip{K}_masks1"].shape[0] == T and int(g[f"clip{K}_masks1"].max()) <= K
        assert g[f"clip{K}_prob1_sub"].shape[0] == K + 1


def test_bounds_catch_a_chunk_only_others_sum():
    """The stem bound of the GPU test refuses an "others" channel summed over the object's chunk only."""
    from test_gpu_many_objects import stem_reference, stem_tolerance
    g = torch.Generator().manual_seed(1)
    K, H, W = 40, 16, 16
    frame = torch.randn((1, 3, H, W), generator=g)
    masks = torch.rand((K, 1, H, W), generator=g)
    for k0, n in object_chunks(K):
        ref = stem_reference(frame, masks, k0, n)
        wrong = stem_reference(frame, masks[k0:k0 + n], 0, n)  # the chunk's masks alone
        assert bool(((wrong - ref).abs() > stem_tolerance(ref, K, False)).any())
        assert bool(((wrong - ref).abs() > stem_tolerance(ref, K, True)).any())


def test_bounds_catch_a_softmax_without_background():
    """The aggregation bound of the GPU test refuses a softmax over the K objects alone."""
    from test_gpu_ops_ragged import aggregate_reference
    g = torch.Generator().manual_seed(2)
    for K in (17, 64, 255):
        p = torch.rand((K, 37), generator=g) * 0.02  # small probabilities: the background dominates
        o, bound, lg = aggregate_reference(p)
        wrong = torch.softmax(lg[1:].float(), 0).double()
        assert bool(((wrong - o[1:]).abs() > bound[1:]).any()), K
