"""Lock-step propagation of several independent clips on ONE GPU.

The reference propagates one sequence per process call (eval_interactive_davis.py:76-83 builds a
fresh processor per sequence); sequences share nothing, which is what shards them over GPUs
(SURVEY.md §8e).  The same independence can be used INSIDE a GPU: the per-frame chain of one clip
is ~70 short dependent kernels whose 1/16- and 1/8-resolution layers have 14-54 row tiles for 132
SMs, so C clips that advance together — same clip length, same interaction history, hence the same
``schedule.PassPlan`` — go through every convolution as one batch of C*K maps (C times the tiles
per launch, one launch instead of C), while the operators whose operands differ per clip (memory
read, skip broadcast, stem gather, aggregation, bank write) are issued per clip on slices of the
batched maps (``engine.PropagationEngine.segment_multi`` / ``encode_memory_multi``).

``LockstepSession([core_0 .. core_{C-1}]).interact([mask_0 ..], idx)`` is C calls of
``InferenceCore.interact(mask_c, idx)`` (reference inference_core.py:219-271): every core ends in
the state its own ``interact`` would have left (prob, masks, np_masks, certain memories,
bank_trace), results are returned per clip.  Each clip keeps its own batched query pass
(``InferenceCore.get_query_kv_buffered``), all of them on one shared side stream.
"""
from __future__ import annotations

import os
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib, ops, schedule
from ._lib import MivosError
from .inference_core import InferenceCore


class _LockStep:
    """The per-frame step of C clips (memory reads -> batched decoder -> aggregation [-> batched
    memorize trunk -> bank writes]) as a captured CUDA graph; the multi-clip analogue of
    ``inference_core._FrameStep``.  What changes per frame lives in device memory the graph reads:
    the C staged frames and query states, and the two int32 scalars (live bank slots, bank frame of
    the memorize) — identical for all clips because they execute the same plan."""

    def __init__(self, net, C: int, K: int, nh: int, nw: int, cap_frames: int):
        eng = net.engine()
        dev = eng.device
        self.net, self.C, self.K, self.nh, self.nw = net, C, K, nh, nw
        self.hw = (nh // 16) * (nw // 16)
        self.cap_frames = cap_frames
        self.frames = torch.zeros((C, 3, nh, nw), dtype=torch.float32, device=dev)
        self.prob = torch.zeros((C, K + 1, 1, nh, nw), dtype=torch.float32, device=dev)
        self.dyn = torch.zeros(4, dtype=torch.int32, device=dev)
        self.states, self.batch = eng.new_query_states(nh, nw, C)
        self.bank_k = torch.empty((C * K, cap_frames * self.hw, 128), dtype=torch.float32, device=dev)
        self.bank_v = torch.empty((C * K, cap_frames * self.hw, 512), dtype=torch.float32, device=dev)
        self.graphs = {}
        self.kernels = {}
        self.use_graph = os.environ.get("MIVOS_GRAPH", "1") != "0"
        # device pointer table (see inference_core._FrameStep): per clip 5 staged operands (sources in dynp[:5C])
        # and K+1 result planes (destinations in dynp[5C:])
        i64 = lambda v: torch.tensor(v, dtype=torch.int64, device=dev)  # noqa: E731
        staged = []
        for c in range(C):
            staged += [self.frames[c], self.batch.kv[c], self.batch.qk[c], self.batch.s8[c], self.batch.s4[c]]
        self.g_fixed = i64([t.data_ptr() for t in staged])
        self.g_bytes_host = [t.numel() * t.element_size() for t in staged]
        self.g_bytes = i64(self.g_bytes_host)
        self.s_fixed = i64([self.prob[c, j].data_ptr() for c in range(C) for j in range(K + 1)])
        self.plane_bytes = nh * nw * 4
        self.s_bytes = i64([self.plane_bytes] * (C * (K + 1)))
        self.dynp = torch.zeros(C * (6 + K), dtype=torch.int64, device=dev)

    @staticmethod
    def get(net, C, K, nh, nw, need_frames):
        cache = net.engine().__dict__.setdefault("_lock_steps", {})
        cap = (need_frames + 15) // 16 * 16
        key = (C, K, nh, nw, cap)
        step = cache.pop(key, None)
        if step is None:
            step = _LockStep(net, C, K, nh, nw, cap)
            while len(cache) >= _LockStep.MAX_CACHED:  # least recently used first out (dict order = use order)
                cache.pop(next(iter(cache)))
        cache[key] = step
        return step

    MAX_CACHED = 2  # lock-step step objects (C*K banks + graphs) kept per network

    def _body(self, memorize: bool):
        eng, C, K = self.net.engine(), self.C, self.K
        ops.copy_segments(self.g_fixed, self.dynp, self.g_bytes, 5 * C, True, max(self.g_bytes_host))
        eng.segment_multi(self.bank_k, self.bank_v, self.cap_frames * self.hw, self.batch, K, C, self.prob,
                          dyn_slots=self.dyn[0:1])
        if memorize:
            kv = eng.encode_memory_multi(self.frames, self.prob[:, 1:])
            h16, w16 = self.nh // 16, self.nw // 16
            # the C*K object banks are contiguous and share the frame slot: one launch
            ops.bank_write(kv, C * K, h16, w16, 0, 128, self.bank_k, self.bank_v, self.cap_frames - 1, dyn_t=self.dyn[1:2])
        ops.copy_segments(self.s_fixed, self.dynp[5 * C:], self.s_bytes, C * (K + 1), False, self.plane_bytes)

    def run(self, frames: Sequence[torch.Tensor], cached, visible: int, m_front: int, memorize: bool, prob_dsts=None, ti: int = 0):
        """`frames[c]` [1,3,nh,nw] (device) and `cached[c]` the QueryState of clip c's frame; `prob_dsts[c]`
        [(K+1),T,1,nh,nw]: the step writes clip c's result planes to prob_dsts[c][:, ti] itself (None: results are
        only left in self.prob[c])."""
        assert visible <= self.cap_frames and m_front < self.cap_frames
        if visible * self.hw < self.net.min_live_slots:  # same rule as the eager path (mivos_memory_read) and torch.topk
            raise MivosError(f"memory_read: {visible * self.hw} live bank slots < top_k {self.net.top_k}")
        C, K = self.C, self.K
        srcs, dsts = [], []
        for c in range(C):
            q = cached[c]
            srcs += [frames[c].data_ptr() if memorize else 0, q.kv.data_ptr(), q.qk.data_ptr(), q.s8.data_ptr(), q.s4.data_ptr()]
            dsts += [prob_dsts[c][j, ti].data_ptr() for j in range(K + 1)] if prob_dsts is not None else [0] * (K + 1)
        ops.store_words(self.dynp, srcs + dsts, self.dyn, (visible * self.hw, m_front))
        if not self.use_graph:
            self._body(memorize)
            return self.prob
        g = self.graphs.get(memorize)
        lib = _lib.load()
        if g is None:
            n0 = lib.mivos_launch_count()
            self._body(memorize)  # eager once: allocates every workspace, sets kernel attributes
            self.kernels[memorize] = lib.mivos_launch_count() - n0
            torch.cuda.current_stream().synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._body(memorize)
            lib.mivos_add_launch_count(-self.kernels[memorize])  # capture issued no work
            self.graphs[memorize] = g
        g.replay()
        lib.mivos_add_launch_count(self.kernels[memorize])
        return self.prob


class LockstepSession:
    def __init__(self, cores: Sequence[InferenceCore]):
        if len(cores) < 1:
            raise MivosError("LockstepSession needs at least one InferenceCore")
        c0 = cores[0]
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
        keys = [core._begin_interaction(m, idx, total_cb if i == 0 else None) for i, (core, m) in enumerate(zip(cores, masks))]
        self._do_pass(keys, idx, True, step_cb)
        self._do_pass(keys, idx, False, step_cb)
        return [core._finish_interaction() for core in cores]

    def _do_pass(self, keys, idx: int, forward: bool, step_cb: Optional[callable]):
        cores = self.cores
        c0 = cores[0]
        C, K, hw = len(cores), c0.k, c0.hw16
        num_certain = c0._certain_bank_k.shape[1] // hw
        plan = schedule.plan_pass(c0.t, c0.interacted, idx, forward, c0.mem_freq, num_certain)
        if not plan.frames:
            return plan.closest_ti
        step = _LockStep.get(c0.prop_net, C, K, c0.nh, c0.nw,
                             schedule.bank_capacity_frames(c0.t, c0.mem_freq, num_certain, plan.total_m))
        for c, core in enumerate(cores):
            o = slice(c * K, (c + 1) * K)
            step.bank_k[o, :num_certain * hw].copy_(core._certain_bank_k)
            step.bank_v[o, :num_certain * hw].copy_(core._certain_bank_v)
        for fp in plan.frames:
            ti = fp.ti
            cached = [core.get_query_kv_buffered(ti, plan.step, plan.closest_ti) for core in cores]
            # the step stages its operands and (unless the frames are fused) writes every clip's prob[:, ti] itself
            frames = [core.get_image_buffered(ti) for core in cores] if fp.memorize else [None] * C
            prob = step.run(frames, cached, fp.visible, fp.m_front, fp.memorize,
                            prob_dsts=None if plan.fuse else [core.prob for core in cores], ti=ti)
            for c, core in enumerate(cores):
                core.bank_trace.append((ti, fp.visible))
                if plan.fuse:
                    core.prob[:, ti] = core.fuse_one_frame(plan.closest_ti, idx, ti, core.prob[:, ti], prob[c], keys[c][0],
                                                           cached[c])
            if step_cb is not None:
                step_cb()
        return plan.closest_ti
