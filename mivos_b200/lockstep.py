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

Clips of an evaluation set differ in length, mem_freq and interaction history, so their pass plans differ.
``LockstepSession(cores, ragged=True)`` takes such a batch (a session without it still requires one plan, as
it always did), and ``interact`` then takes one interaction frame per clip.  A batch whose plans differ runs
RAGGED (``_run_ragged_pass``): every clip executes its own ``schedule.PassPlan``; at the start of a pass the
clips are ordered longest pass first, so the clips that still have a frame at a tick — and those that memorize
— are a prefix, and a tick runs the step over the leading rows of its C-clip banks and buffers.  Each clip's
live slot count and memorize frame are per-clip device counters of the step, read by the per-set forms of the
memory read and of the bank write.  Clips that share one plan keep the path above unchanged.

``LockstepSession(cores, mixed_objects=True)`` (ragged, and 1 to 16 objects per clip) also takes clips of different
object counts.  The step is then sized for the clips' total object count: position p of the pass order owns bank
rows and object maps [first[p], first[p+1]) and the packed result planes [first[p] + p, first[p+1] + p + 1) (its
background, then its objects).  `first` goes into the step's pointer table with the counters, and the operators
whose operands differ per clip take it in their object-group forms.  Clips of one object count run exactly as in a
ragged session.
"""
from __future__ import annotations

from typing import List, Sequence, Union

import numpy as np
import torch

from . import schedule
from ._lib import MivosError
from .engine import CHUNK_OBJECTS
from .frame_step import FrameStep
from .inference_core import InferenceCore, run_pass


class LockstepSession:
    def __init__(self, cores: Sequence[InferenceCore], ragged: bool = False, mixed_objects: bool = False):
        """`ragged`: the clips may differ in length, mem_freq, mem_profile and interaction history (each runs its
        own pass plan); without it they must share one plan.  `mixed_objects` (implies `ragged`): the clips may also
        differ in object count (1 to 16 each)."""
        if len(cores) < 1:
            raise MivosError("LockstepSession needs at least one InferenceCore")
        ragged = ragged or mixed_objects
        c0 = cores[0]
        for i, c in enumerate(cores):
            if c.k > CHUNK_OBJECTS:
                raise MivosError(f"LockstepSession: clip {i} has {c.k} objects; lock-step clips take at most "
                                 f"{CHUNK_OBJECTS} (more objects run in object chunks, which only InferenceCore does): "
                                 "run the clip separately")
            if not mixed_objects:
                break
        for i, c in enumerate(cores[1:], 1):
            if c.prop_net is not c0.prop_net:
                raise MivosError(f"lock-step clips must share one network: clip {i} has another")
            if c.device != c0.device:
                raise MivosError(f"lock-step clips must share one device: clip {i} is on {c.device}, clip 0 on {c0.device}")
            if c.k != c0.k and not mixed_objects:
                raise MivosError(f"lock-step clips must have the same object count: clip {i} has {c.k}, clip 0 {c0.k}; "
                                 "group the clips by object count, one session per group")
            if (c.nh, c.nw) != (c0.nh, c0.nw):
                raise MivosError(f"lock-step clips must have the same padded size: clip {i} is {c.nh}x{c.nw}, clip 0 "
                                 f"{c0.nh}x{c0.nw}")
            if not ragged and not (c.t == c0.t and c.mem_freq == c0.mem_freq and c.interacted == c0.interacted):
                raise MivosError("lock-step clips must share the length, mem_freq and interaction history (they "
                                 "execute one PassPlan), unless the session is made with ragged=True")
        self.ragged = ragged
        self.mixed_objects = mixed_objects
        self.cores: List[InferenceCore] = list(cores)
        # the clips share ONE network, hence one query-pass workspace (engine.ws_q): their batched query
        # passes must be stream-ordered among themselves, so they all run on the first clip's side stream
        for c in cores[1:]:
            c._qstream = c0._qstream

    def interact(self, masks: Sequence[torch.Tensor], idx: Union[int, Sequence[int]], total_cb=None,
                 step_cb=None) -> List[np.ndarray]:
        """C x InferenceCore.interact(mask_c, idx_c); `idx` is one frame for all clips or, in a ragged session, one per
        clip.  `total_cb(n)` / `step_cb()` count lock-step ticks (n = ticks of the two passes, called once; one step_cb
        per tick)."""
        cores = self.cores
        if len(masks) != len(cores):
            raise MivosError(f"{len(cores)} clips but {len(masks)} masks")
        idxs = [idx] * len(cores) if isinstance(idx, int) else [int(i) for i in idx]
        if len(idxs) != len(cores):
            raise MivosError(f"{len(cores)} clips but {len(idxs)} interaction frames")
        if not self.ragged and any(i != idxs[0] for i in idxs):
            raise MivosError("one interaction frame per clip needs a session made with ragged=True")
        c0 = cores[0]
        one_plan = all(i == idxs[0] for i in idxs) and all(
            c.t == c0.t and c.mem_freq == c0.mem_freq and c.interacted == c0.interacted and c.k == c0.k for c in cores)
        if one_plan:  # every clip executes the same PassPlan
            keys = [core._begin_interaction(m, idxs[0], total_cb if i == 0 else None)[0]
                    for i, (core, m) in enumerate(zip(cores, masks))]
            run_pass(cores, keys, idxs[0], True, step_cb)
            run_pass(cores, keys, idxs[0], False, step_cb)
            return [core._finish_interaction() for core in cores]
        keys = [core._begin_interaction(m, i)[0] for core, m, i in zip(cores, masks, idxs)]
        setups = [_ragged_pass_setup(cores, idxs, forward) for forward in (True, False)]
        ticks = sum(max(len(p.frames) for p in plans) for plans, _, _ in setups)
        if total_cb is not None and ticks > 0:
            total_cb(ticks)
        for plans, order, step in setups:
            if step is not None:
                _run_ragged_pass(cores, keys, idxs, plans, order, step, step_cb)
        return [core._finish_interaction() for core in cores]


def _ragged_pass_setup(cores, idxs, forward):
    """Per-clip plans of one pass, the clip order (schedule.pass_order) and the ragged step that serves them (None:
    no clip has a frame in this pass).  The step's banks are sized for the largest capacity over the clips."""
    c0 = cores[0]
    K, hw = c0.k, c0.hw16
    certain = [core._certain_bank_k.shape[1] // hw for core in cores]
    plans = [schedule.plan_pass(core.t, core.interacted, i, forward, core.mem_freq, n)
             for core, i, n in zip(cores, idxs, certain)]
    order = schedule.pass_order(plans)
    if not plans[order[0]].frames:
        return plans, order, None
    cap = max(schedule.bank_capacity_frames(core.t, core.mem_freq, n, p.total_m)
              for core, n, p in zip(cores, certain, plans))
    if any(c.k != K for c in cores):  # mixed object counts: bank rows and planes for the clips' total
        step = FrameStep.get(c0.prop_net, len(cores), max(c.k for c in cores), c0.nh, c0.nw, cap, 0, ragged=True,
                             maps=sum(c.k for c in cores))
    else:
        step = FrameStep.get(c0.prop_net, len(cores), K, c0.nh, c0.nw, cap, 0, ragged=True)
    return plans, order, step


def _run_ragged_pass(cores, keys, idxs, plans, order, step, step_cb):
    """One pass of every clip, each on its own plan, in lock-step ticks: at tick i the first n clips of `order` have a
    frame, the first n_mem of them memorize (schedule.tick_prefixes).  Bank rows follow the position in `order`."""
    K, hw = cores[0].k, cores[0].hw16
    mixed = step.maps is not None
    # object maps of position p: [first[p], first[p+1]) — p * K with one object count
    ks = [cores[c].k for c in order]
    first = [0]
    for k in ks:
        first.append(first[-1] + k)
    # every clip's certain memories into the bank rows of its position (:146-151); the step's banks are only
    # written by this session's ticks until the pass ends, so the copies of both passes happen at their start
    for p, c in enumerate(order):
        n = cores[c]._certain_bank_k.shape[1]
        step.bank_k[first[p]:first[p + 1], :n].copy_(cores[c]._certain_bank_k)
        step.bank_v[first[p]:first[p + 1], :n].copy_(cores[c]._certain_bank_v)
    graph = cores[0].use_graph
    for i in range(len(plans[order[0]].frames)):
        n, n_mem = schedule.tick_prefixes(plans, order, i)
        act = order[:n]
        fps = [plans[c].frames[i] for c in act]
        cached = [cores[c].get_query_kv_buffered(fp.ti, plans[c].step, plans[c].closest_ti) for c, fp in zip(act, fps)]
        frames = [cores[c].get_image_buffered(fp.ti) if p < n_mem else None for p, (c, fp) in enumerate(zip(act, fps))]
        prob = step.run_ragged(frames, cached, [fp.visible for fp in fps], [fp.m_front for fp in fps], n_mem,
                               [None if plans[c].fuse else cores[c]._results() for c in act], [fp.ti for fp in fps], graph,
                               ks=ks if mixed else None)
        for p, (c, fp) in enumerate(zip(act, fps)):
            core, plan = cores[c], plans[c]
            core.bank_trace.append((fp.ti, fp.visible))
            if plan.fuse:  # :190-194
                # the clip's planes: prob[p] [K+1,...], or its packed range (background, then its objects)
                planes = prob[first[p] + p:first[p + 1] + p + 1] if mixed else prob[p]
                core._set_frame(fp.ti, core.fuse_one_frame(plan.closest_ti, idxs[c], fp.ti, core._frame(fp.ti), planes,
                                                           keys[c], cached[p]))
        if step_cb is not None:
            step_cb()
