"""Lock-step propagation of several independent clips on ONE GPU.

The reference propagates one sequence per process call (eval_interactive_davis.py:76-83 builds a
fresh processor per sequence); sequences share nothing, which is what shards them over GPUs
(SURVEY.md §8e).  The same independence can be used INSIDE a GPU: the per-frame chain of one clip
is ~70 short dependent kernels whose 1/16- and 1/8-resolution layers have 14-54 row tiles for 132
SMs, so C clips that advance together — same clip length, same interaction history, hence the same
``schedule.PassPlan`` — go through every convolution as one batch of C*K maps (C times the tiles
per launch, one launch instead of C), while the operators whose operands differ per clip (memory
read, skip broadcast, stem gather, aggregation) take the C clips as groups of one launch.  The step
is ``frame_step.FrameStep`` with C clips and the pass loop is ``inference_core.run_pass`` over the C
cores: the code a single ``InferenceCore`` runs with C = 1.

``LockstepSession([core_0 .. core_{C-1}]).interact([mask_0 ..], idx)`` is C calls of
``InferenceCore.interact(mask_c, idx)`` (reference inference_core.py:219-271): every core ends in
the state its own ``interact`` would have left (prob, masks, np_masks, certain memories,
bank_trace), results are returned per clip.  Each clip keeps its own batched query pass
(``InferenceCore.get_query_kv_buffered``), all of them on one shared side stream.  The first
core's ``use_graph`` decides between graph replay and eager launches.
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np
import torch

from ._lib import MivosError
from .engine import CHUNK_OBJECTS
from .inference_core import InferenceCore, run_pass


class LockstepSession:
    def __init__(self, cores: Sequence[InferenceCore]):
        if len(cores) < 1:
            raise MivosError("LockstepSession needs at least one InferenceCore")
        c0 = cores[0]
        if c0.k > CHUNK_OBJECTS:
            raise MivosError(f"LockstepSession: {c0.k} objects per clip; lock-step clips take at most {CHUNK_OBJECTS} "
                             "(more objects run in object chunks, which only InferenceCore does): run the clips separately")
        for c in cores[1:]:
            same = (c.prop_net is c0.prop_net and c.device == c0.device and c.k == c0.k and c.t == c0.t and c.nh == c0.nh
                    and c.nw == c0.nw and c.mem_freq == c0.mem_freq and c.interacted == c0.interacted)
            if not same:
                raise MivosError("lock-step clips must share the network, device, object count, length, padded size, "
                                 "mem_freq and interaction history (they execute one PassPlan); run the others separately")
        self.cores: List[InferenceCore] = list(cores)
        # the clips share ONE network, hence one query-pass workspace (engine.ws_q): their batched query
        # passes must be stream-ordered among themselves, so they all run on the first clip's side stream
        for c in cores[1:]:
            c._qstream = c0._qstream

    def interact(self, masks: Sequence[torch.Tensor], idx: int, total_cb=None, step_cb=None) -> List[np.ndarray]:
        """C x InferenceCore.interact(mask_c, idx).  `total_cb(n)` / `step_cb()` count frames per clip
        step (n = frames of the two passes; one step_cb per lock-step frame)."""
        cores = self.cores
        if len(masks) != len(cores):
            raise MivosError(f"{len(cores)} clips but {len(masks)} masks")
        keys = [core._begin_interaction(m, idx, total_cb if i == 0 else None)[0] for i, (core, m) in enumerate(zip(cores, masks))]
        run_pass(cores, keys, idx, True, step_cb)
        run_pass(cores, keys, idx, False, step_cb)
        return [core._finish_interaction() for core in cores]
