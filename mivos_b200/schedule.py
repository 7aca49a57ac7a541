"""Bank bookkeeping of one propagation pass as pure host arithmetic (no tensors, no device).

``InferenceCore.do_pass`` (reference inference_core.py:122-200) interleaves this bookkeeping with
the network calls; here it is separated out so that (a) it is unit-tested on the CPU against the
oracle's trace, and (b) the single-clip driver (``InferenceCore.do_pass``) and the lock-step
multi-clip driver (``lockstep.LockstepSession``) execute the SAME plan.

Rules restated (reference lines):
  * the pass runs from the interacted frame towards the closest other interacted frame, or the clip
    end (:128-141); ``total_m`` bank frames are needed (:136-141);
  * bank slot ``m_front`` is overwritten by every propagated frame except the last one of the pass
    (:177-179); the slot is *committed* (``m_front += 1``) when the frame is ``mem_freq`` or more
    frames away from the last committed one (:180-186);
  * a frame sees ``m_front`` slots when the previous frame's memory was committed (or at the start
    of the pass) and ``m_front + 1`` — the temporary slot included — otherwise (:166-171);
  * frames are fused with the previous pass's result when the pass is bounded by another
    interaction (:190-194).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Iterable, List


@dataclass(frozen=True)
class FramePlan:
    ti: int          # frame index
    visible: int     # bank frames the memory read sees
    m_front: int     # bank frame the memorize of this frame writes (when `memorize`)
    memorize: bool   # False only for the last frame of the pass


@dataclass
class PassPlan:
    idx: int
    forward: bool
    closest_ti: int
    total_m: int     # bank frames the pass needs (reference :136-141)
    fuse: bool
    frames: List[FramePlan] = field(default_factory=list)

    @property
    def step(self) -> int:
        return 1 if self.forward else -1


def plan_pass(t: int, interacted: Iterable[int], idx: int, forward: bool, mem_freq: int, num_certain: int) -> PassPlan:
    interacted = set(interacted)
    if forward:
        closest_ti = min([ti for ti in interacted if ti > idx] + [t])
        total_m = (closest_ti - idx - 1) // mem_freq + 1 + num_certain
        rng, end = range(idx + 1, closest_ti), closest_ti - 1
    else:
        closest_ti = max([ti for ti in interacted if ti < idx] + [-1])
        total_m = (idx - closest_ti - 1) // mem_freq + 1 + num_certain
        rng, end = range(idx - 1, closest_ti, -1), closest_ti + 1
    plan = PassPlan(idx=idx, forward=forward, closest_ti=closest_ti, total_m=total_m,
                    fuse=(closest_ti != t) and (closest_ti != -1))
    m_front, prev_in_mem, last_ti = num_certain, True, idx
    for ti in rng:
        visible = m_front if prev_in_mem else m_front + 1
        memorize = ti != end
        plan.frames.append(FramePlan(ti, visible, m_front, memorize))
        if memorize:
            if abs(ti - last_ti) >= mem_freq:
                m_front += 1
                last_ti = ti
                prev_in_mem = True
            else:
                prev_in_mem = False
    return plan


INTERACTION_BUDGET = 16  # certain memories a clip's bank is sized for before it has to grow


def bank_capacity_frames(t: int, mem_freq: int, num_certain: int, total_m: int) -> int:
    """Bank frames to allocate so that the bank pointers (and the CUDA graphs captured over them)
    stay valid across the passes of a clip: the longest pass of the clip plus a FIXED budget of
    interactions.  The result does not depend on the current number of certain memories (as long as it
    is within the budget), so every pass and every session over clips of this length shares one entry
    of the frame-step cache."""
    return max(total_m, (t - 2) // mem_freq + 2 + INTERACTION_BUDGET)


def pass_order(plans: List[PassPlan]) -> List[int]:
    """Clips of one lock-step pass, longest pass first (stable on ties).  In this order the clips that still have a
    frame at tick i are a prefix (those with more than i frames), and so are the clips that memorize at tick i: a
    clip skips the memorize only on its last frame, so they are those with more than i + 1 frames."""
    return sorted(range(len(plans)), key=lambda c: -len(plans[c].frames))


def tick_prefixes(plans: List[PassPlan], order: List[int], i: int):
    """(clips with a frame at tick i, clips memorizing at tick i), both prefixes of `order`."""
    n = sum(1 for c in order if len(plans[c].frames) > i)
    n_mem = sum(1 for c in order[:n] if plans[c].frames[i].memorize)
    return n, n_mem
