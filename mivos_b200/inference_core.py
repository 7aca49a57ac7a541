"""Drop-in ``InferenceCore`` (reference: inference_core.py:17-292).

Same constructor, methods, callbacks and public attributes (``prob masks np_masks images pad k t
h w nh nw interacted certain_mem_k certain_mem_v``) so eval_interactive_davis.py / davis_processor.py
/ interactive_gui.py run unchanged.  What differs is where the state lives and how a frame is
processed:

  * the memory bank is slot-major (BANK layout) and written in place by the memorize conv stack —
    no torch.cat, no [K,C,T,H,W] transposes on the hot loop (reference :146-151, :178);
  * query features are cached per frame index as resident HALO maps (reference :110-120);
  * one propagated frame = query encoder -> fused memory read -> decoder -> 4x upsample + sigmoid
    + aggregate_wbg (one kernel) -> memorize; the per-frame argmax loop (:259-260), unpad and the
    u8 conversion are a single kernel over the whole clip.

Bank bookkeeping (temporary slot, commit every mem_freq frames, last frame never memorised)
follows inference_core.py:132-186 line by line.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

import os

from . import _lib, ops, schedule
from .engine import QueryState
from .tensor_util import pad_divide_by


class _FrameStep:
    """One propagated frame (query encoder -> memory read -> decoder -> aggregate [-> memorize]) as
    a captured CUDA graph.  Everything that changes from frame to frame lives in device memory the
    graph reads: the frame is staged into `frame`, the live bank size and the bank slot of the
    memorize are the int32 scalars `dyn` (mivos_store_i32 writes them from launch arguments), the
    result lands in `prob`.  The query-side features of the frame come from the batched query pass
    (InferenceCore.get_query_kv_buffered) and are staged into `qs`.  One graph with and one
    without the memorize serve every frame of
    every pass while the bank grows, so the ~130 kernel launches of a frame cost one graph launch
    on the host.  Instances (with their bank buffers) are cached on the network's engine, keyed by
    (objects, padded size, bank capacity), and shared by successive InferenceCore objects — the
    reference also shares the networks between sessions (eval_interactive_davis.py:83)."""

    def __init__(self, net, K: int, nh: int, nw: int, cap_frames: int, lane: int = 0):
        eng = net.engine()
        dev = eng.device
        self.net, self.K, self.nh, self.nw, self.lane = net, K, nh, nw, lane
        self.hw = (nh // 16) * (nw // 16)
        self.cap_frames = cap_frames
        self.frame = torch.zeros((1, 3, nh, nw), dtype=torch.float32, device=dev)
        self.prob = torch.zeros((K + 1, 1, nh, nw), dtype=torch.float32, device=dev)
        self.dyn = torch.zeros(4, dtype=torch.int32, device=dev)
        self.qs = eng.new_query_state(nh, nw)
        self.bank_k = torch.empty((K, cap_frames * self.hw, 128), dtype=torch.float32, device=dev)
        self.bank_v = torch.empty((K, cap_frames * self.hw, 512), dtype=torch.float32, device=dev)
        self.graphs = {}
        self.kernels = {}  # kernels per replay, for mivos_launch_count accounting
        # Device pointer table of the step (mivos_copy_segments): the graph STAGES the frame's operands itself —
        # frame, cached query features kv / qk / s8 / s4: source pointers in dynp[0:5] — and DELIVERS the K+1 result
        # planes to InferenceCore.prob[:, ti] (destination pointers in dynp[5:]); per frame the host writes the table
        # and the two bank counters with ONE small launch (mivos_store_words) and replays the graph: no eager copy.
        staged = [self.frame, self.qs.kv, self.qs.qk, self.qs.s8, self.qs.s4]
        i64 = lambda v: torch.tensor(v, dtype=torch.int64, device=dev)  # noqa: E731
        self.g_fixed = i64([t.data_ptr() for t in staged])
        self.g_bytes_host = [t.numel() * t.element_size() for t in staged]
        self.g_bytes = i64(self.g_bytes_host)
        self.s_fixed = i64([self.prob[j].data_ptr() for j in range(K + 1)])
        self.plane_bytes = nh * nw * 4
        self.s_bytes = i64([self.plane_bytes] * (K + 1))
        self.dynp = torch.zeros(5 + K + 1, dtype=torch.int64, device=dev)

    MAX_CACHED = 4  # step objects (bank + query staging + graphs) kept per network, least recently used first out

    @staticmethod
    def get(net, K, nh, nw, need_frames, lane: int = 0):
        eng = net.engine()
        cache = eng.__dict__.setdefault("_frame_steps", {})
        cap = (need_frames + 15) // 16 * 16
        key = (K, nh, nw, cap, lane)
        step = cache.pop(key, None)
        if step is None:
            step = _FrameStep(net, K, nh, nw, cap, lane)
            while len(cache) >= _FrameStep.MAX_CACHED:  # evict the least recently used entry (dict order = use order)
                cache.pop(next(iter(cache)))
        cache[key] = step  # (re)insert as most recently used
        return step

    def _body(self, memorize: bool):
        net = self.net
        with net.engine().lane(self.lane):
            ops.copy_segments(self.g_fixed, self.dynp, self.g_bytes, 5, True, max(self.g_bytes_host))
            net.segment_resident(self.bank_k, self.bank_v, self.cap_frames * self.hw, self.qs, self.K, prob_out=self.prob,
                                 dyn_slots=self.dyn[0:1])
            if memorize:
                net.memorize_resident(self.frame, self.prob[1:], self.bank_k, self.bank_v, self.cap_frames - 1,
                                      dyn_slot=self.dyn[1:2])
            ops.copy_segments(self.s_fixed, self.dynp[5:], self.s_bytes, self.K + 1, False, self.plane_bytes)

    def run(self, frame, qs_cached: QueryState, visible_frames: int, m_front: int, memorize: bool, prob_dst=None, ti: int = 0):
        """`frame` [1,3,nh,nw] and `qs_cached` on the device; `prob_dst` [(K+1),T,1,nh,nw]: the step writes its result
        planes to prob_dst[:, ti] itself (None: the result is only left in self.prob, e.g. for fuse_one_frame)."""
        assert visible_frames <= self.cap_frames and m_front < self.cap_frames
        if visible_frames * self.hw < self.net.min_live_slots:  # same rule as the eager path (mivos_memory_read) and torch.topk
            raise _lib.MivosError(f"memory_read: {visible_frames * self.hw} live bank slots < top_k {self.net.top_k}")
        srcs = [frame.data_ptr() if memorize else 0, qs_cached.kv.data_ptr(), qs_cached.qk.data_ptr(),
                qs_cached.s8.data_ptr(), qs_cached.s4.data_ptr()]
        dsts = [prob_dst[j, ti].data_ptr() for j in range(self.K + 1)] if prob_dst is not None else [0] * (self.K + 1)
        ops.store_words(self.dynp, srcs + dsts, self.dyn, (visible_frames * self.hw, m_front))
        g = self.graphs.get(memorize)
        if g is None:
            # first use: run eagerly once (allocates every workspace, sets kernel attributes), then capture
            lib = _lib.load()
            n0 = lib.mivos_launch_count()
            self._body(memorize)
            self.kernels[memorize] = lib.mivos_launch_count() - n0
            torch.cuda.current_stream().synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._body(memorize)
            lib.mivos_add_launch_count(-self.kernels[memorize])  # capture issued no work
            self.graphs[memorize] = g
        g.replay()
        _lib.load().mivos_add_launch_count(self.kernels[memorize])
        return self.prob, self.qs


class InferenceCore:
    def __init__(self, prop_net, fuse_net, images, num_objects, mem_profile=0, mem_freq=5, device="cuda:0"):
        self.device = torch.device(device)
        _lib.require_cuda_device(self.device, "mivos_b200.InferenceCore")
        self.prop_net = prop_net.to(self.device, non_blocking=True)
        if fuse_net is not None:
            self.fuse_net = fuse_net.to(self.device, non_blocking=True)
        self.mem_profile = mem_profile
        self.mem_freq = mem_freq

        # Same buffer policy table as the reference (:44-63).  Results always live on the device
        # here (a 480p prob volume is 1.66 MB per frame per object); the
        # query-feature cache honours q_buf_size, image staging honours data_dev / i_buf_size.
        if mem_profile == 0:
            self.data_dev, self.q_buf_size, self.i_buf_size = self.device, 105, -1
        elif mem_profile == 1:
            self.data_dev, self.q_buf_size, self.i_buf_size = torch.device("cpu"), 105, 105
        elif mem_profile == 2:
            self.data_dev, self.q_buf_size, self.i_buf_size = torch.device("cpu"), 3, 3
        else:
            self.data_dev, self.q_buf_size, self.i_buf_size = torch.device("cpu"), 1, 1
        self.result_dev = self.device

        t = images.shape[1]
        h, w = images.shape[-2:]
        self.k = num_objects
        images = images.float()
        self.images, self.pad = pad_divide_by(images, 16, images.shape[-2:])  # :71
        nh, nw = self.images.shape[-2:]
        if self.data_dev.type == "cpu":
            self.images = self.images.cpu().contiguous()
            if not self.images.is_pinned():
                self.images = self.images.pin_memory()  # async H2D per frame (get_image_buffered)
        else:
            self.images = self.images.to(self.device).contiguous()

        self.masks = torch.zeros((t, 1, nh, nw), dtype=torch.uint8, device=self.result_dev)  # :77
        # result masks cross PCIe into ONE pinned staging buffer (async D2H at link rate instead of a
        # pageable copy); interact() hands the caller a fresh array copied from it, as the reference's
        # `.cpu().numpy()` does (:269)
        self._masks_host = torch.zeros((t, h, w), dtype=torch.uint8).pin_memory()
        self.np_masks = np.zeros((t, h, w), dtype=np.uint8)
        self.prob = torch.zeros((self.k + 1, t, 1, nh, nw), dtype=torch.float32, device=self.result_dev)  # :81
        self.prob[0] = 1e-7  # :82

        self.t, self.h, self.w = t, h, w
        self.nh, self.nw = nh, nw
        self.kh, self.kw = nh // 16, nw // 16
        self.hw16 = self.kh * self.kw

        self.query_buf: Dict[int, QueryState] = {}
        # Batched QueryState allocations (states, batch) of QUERY_CHUNK frames each.  The cache the
        # reference fills lazily (:110-120) is allocated HERE, with the other per-session buffers
        # (prob, masks — reference :81-84), so that interact() never calls cudaMalloc: enough chunks
        # for min(t, q_buf_size) cached frames plus the one being refilled after a flush.
        chunk = max(1, min(self.QUERY_CHUNK, self.q_buf_size))
        n_chunks = (min(t, self.q_buf_size + 1) + chunk - 1) // chunk + 1
        eng = self.prop_net.engine()
        self._query_pool = [eng.new_query_states(nh, nw, chunk) for _ in range(n_chunks)]
        self._query_chunks = []  # allocations backing query_buf
        self._query_ready = {}   # frame idx -> event recorded after its batched query pass
        # ONE side stream per network: the batched query passes of every session over this network write the
        # engine's single query-pass workspace (engine.ws_q), so they must be stream-ordered among themselves
        if eng.__dict__.get("_qstream") is None:
            eng._qstream = torch.cuda.Stream(device=self.device)
        self._qstream = eng._qstream
        self.image_buf: Dict[int, torch.Tensor] = {}
        # device staging slots for frames uploaded from the host clip (mem_profile >= 1), allocated
        # once so that interact() does not call cudaMalloc per frame
        self._image_slots = None
        if self.data_dev != self.device:
            self._image_slots = torch.empty((min(t, max(self.i_buf_size, 0) + 2), 1, 3, nh, nw), dtype=torch.float32,
                                            device=self.device)
        self.interacted = set()

        self.certain_mem_k = None  # reference layout [K,128,n,kh,kw], kept for attribute compatibility
        self.certain_mem_v = None
        self._certain_bank_k = None  # BANK layout [K, n*hw16, 128]
        self._certain_bank_v = None
        self._bank_k = None
        self._bank_v = None
        self._masks_unpadded = torch.zeros((t, h, w), dtype=torch.uint8, device=self.device)
        self._fuse_planes = None
        self.bank_trace = []  # (frame, visible bank frames) per propagated frame, for plumbing tests
        # CUDA-graph replay of the per-frame step (MIVOS_GRAPH=0 falls back to eager launches)
        self.use_graph = os.environ.get("MIVOS_GRAPH", "1") != "0"
        # forward and backward pass of one interaction as two concurrent lanes (MIVOS_BIDIR=0: one after the other)
        self.overlap_passes = os.environ.get("MIVOS_BIDIR", "1") != "0"
        self._lane_stream = None
        self._pass_streams = ()  # streams of the passes in flight (two while the passes of an interaction overlap)

    # ------------------------------------------------------------------ buffers (:96-120)
    def get_image_buffered(self, idx):
        if self.data_dev == self.device:
            return self.images[:, idx]
        if idx not in self.image_buf:
            if len(self.image_buf) > self.i_buf_size:  # wholesale flush, like the reference (:101-103)
                self.image_buf = {}
                # staged frames may still be read by the batched query pass on the side stream
                torch.cuda.current_stream(self.device).wait_stream(self._qstream)
            slot = self._image_slots[len(self.image_buf)]
            slot.copy_(self.images[:, idx], non_blocking=True)  # pinned host -> preallocated device slot
            self.image_buf[idx] = slot
        return self.image_buf[idx]

    QUERY_CHUNK = 8  # frames per batched query pass

    def _issue_query_chunk(self, want):
        """Encode the (sorted) frames `want` in one batched query pass on the side stream."""
        n = len(want)
        entry = next((e for e in self._query_pool if len(e[0]) >= n), None)
        if entry is not None:
            self._query_pool.remove(entry)
        else:
            entry = self.prop_net.engine().new_query_states(self.nh, self.nw, max(n, min(self.QUERY_CHUNK, self.q_buf_size)))
        states, batch = entry
        if len(states) > n:  # a short tail chunk uses the first n frames of the allocation
            states, batch = states[:n], batch.first(n)
        if self.data_dev == self.device and want[-1] - want[0] == n - 1:
            frames = self.images[0, want[0]:want[0] + n]  # contiguous device view, no copy
        elif self.data_dev == self.device:
            frames = torch.stack([self.images[0, j] for j in want], 0)
        else:
            # host clip: upload through the staging slots (each frame crosses PCIe once; memorize
            # reads the same slot later).  No wholesale flush may happen while the list is built,
            # or a slot handed out earlier in this loop would be overwritten.
            missing = [j for j in want if j not in self.image_buf]
            if len(self.image_buf) + len(missing) > self.i_buf_size + 1:
                self.image_buf = {}
                torch.cuda.current_stream(self.device).wait_stream(self._qstream)
            first = len(self.image_buf)
            slots = [self.get_image_buffered(j) for j in want]
            if len(missing) == n and want[-1] - want[0] == n - 1:
                frames = self._image_slots[first:first + n, 0]  # freshly staged, contiguous: no copy
            else:
                frames = torch.stack([sl[0] for sl in slots], 0)
        cur = torch.cuda.current_stream(self.device)
        self._qstream.wait_stream(cur)  # frame uploads / earlier readers of the pooled buffers come first
        for st in self._pass_streams:   # overlapped passes: the OTHER lane may still read recycled pooled buffers
            if st is not cur:
                self._qstream.wait_stream(st)
        with torch.cuda.stream(self._qstream):
            self.prop_net.encode_query_batch_resident(frames, batch)
            ready = torch.cuda.Event()
            ready.record(self._qstream)
        frames.record_stream(self._qstream)
        self._query_chunks.append(entry)
        for j, st in zip(want, states):
            self.query_buf[j] = st
            self._query_ready[j] = ready

    def get_query_kv_buffered(self, idx, step: int = 1, stop: Optional[int] = None) -> QueryState:
        """Query-side features of frame idx (reference :110-120: computed once per frame index and
        cached; wholesale flush when the cache exceeds q_buf_size).  The features depend on the
        frames only, so the frames the pass will visit next (idx, idx+step, ... before `stop`) are
        encoded QUERY_CHUNK at a time in one batched pass — batching is what fills the GPU on the
        1/8- and 1/16-resolution layers — on a side stream, one chunk ahead of the frame loop, so the
        pass overlaps the sequential part (memory read, decoder tail, memorize) of earlier frames."""
        chunk = max(1, min(self.QUERY_CHUNK, self.q_buf_size))
        lookahead = 2 * chunk if self.q_buf_size >= 2 * self.QUERY_CHUNK else 1
        j, covered = idx, 0
        while covered < lookahead and 0 <= j < self.t and (stop is None or j != stop):
            if j in self.query_buf:
                j += step
                covered += 1
                continue
            if len(self.query_buf) > self.q_buf_size and j == idx:
                self._query_pool.extend(self._query_chunks)  # flush wholesale like :114-115, keep the memory
                self.query_buf, self._query_chunks, self._query_ready = {}, [], {}
            want = []
            while len(want) < chunk and 0 <= j < self.t and (stop is None or j != stop):
                if j not in self.query_buf:
                    want.append(j)
                j += step
            covered += len(want)
            want.sort()
            self._issue_query_chunk(want)
        torch.cuda.current_stream(self.device).wait_event(self._query_ready[idx])
        return self.query_buf[idx]

    # ------------------------------------------------------------------ one pass (:122-200)
    def _pass_setup(self, idx, forward, lane: int = 0):
        """Plan of one pass (:128-141), its frame-step object / bank (lane 0 or 1), certain memories copied in
        (:146-151)."""
        K, hw = self.k, self.hw16
        num_certain = self._certain_bank_k.shape[1] // hw
        # the bank bookkeeping of the pass (:128-141, :166-186) is host arithmetic: schedule.plan_pass
        plan = schedule.plan_pass(self.t, self.interacted, idx, forward, self.mem_freq, num_certain)
        step = None
        if not plan.frames:
            return plan, None, None, None
        if self.use_graph:
            # bank sized for the longest pass of this clip plus a fixed interaction budget, so the bank
            # pointers (and with them the captured graphs) stay valid across passes and sessions
            step = _FrameStep.get(self.prop_net, K, self.nh, self.nw,
                                  schedule.bank_capacity_frames(self.t, self.mem_freq, num_certain, plan.total_m), lane)
            bank_k, bank_v = step.bank_k, step.bank_v
        else:
            need = plan.total_m * hw
            if self._bank_k is None or self._bank_k.shape[1] < need:
                self._bank_k = torch.empty((K, need, 128), dtype=torch.float32, device=self.device)
                self._bank_v = torch.empty((K, need, 512), dtype=torch.float32, device=self.device)
            bank_k, bank_v = self._bank_k, self._bank_v
        bank_k[:, :num_certain * hw].copy_(self._certain_bank_k)
        bank_v[:, :num_certain * hw].copy_(self._certain_bank_v)
        return plan, step, bank_k, bank_v

    def _pass_frame(self, plan, step, bank_k, bank_v, fp, key_k, idx, trace):
        """One propagated frame of a pass (:165-194) on the current stream."""
        K, hw, ti = self.k, self.hw16, fp.ti
        trace.append((ti, fp.visible))
        qs = self.get_query_kv_buffered(ti, plan.step, plan.closest_ti)  # :172
        if step is not None:
            # the graph stages the operands and (unless the frame is fused) writes prob[:, ti] itself  # :173-179, :194
            frame = self.get_image_buffered(ti) if fp.memorize else None
            out_mask, qs = step.run(frame, qs, fp.visible, fp.m_front, fp.memorize,
                                    prob_dst=None if plan.fuse else self.prob, ti=ti)
        else:
            _, out_mask = self.prop_net.segment_resident(bank_k, bank_v, fp.visible * hw, qs, K)  # :173-175
            if fp.memorize:  # :177-179
                self.prop_net.memorize_resident(self.get_image_buffered(ti), out_mask[1:], bank_k, bank_v, fp.m_front)
        if plan.fuse:  # :190-194
            self.prob[:, ti] = self.fuse_one_frame(plan.closest_ti, idx, ti, self.prob[:, ti], out_mask, key_k, qs)
        elif step is None:
            self.prob[:, ti] = out_mask

    def do_pass(self, key_k, key_v, idx, forward=True, step_cb=None):
        plan, step, bank_k, bank_v = self._pass_setup(idx, forward)
        for fp in plan.frames:
            self._pass_frame(plan, step, bank_k, bank_v, fp, key_k, idx, self.bank_trace)
            if step_cb is not None:
                step_cb()
        return plan.closest_ti

    def _do_passes_overlapped(self, key_k, key_v, idx, step_cb=None):
        """The forward and the backward pass of one interaction are independent until the argmax
        (inference_core.py:255-256): they run here as two LANES — own frame-step graphs, bank, workspace
        (engine.lane(1)) and CUDA stream — issued frame by frame in alternation, so the kernels of one
        pass fill the SMs the other's latency-bound chain leaves idle.  Each pass executes exactly the
        launches of do_pass in the same order: results are bit-identical to the sequential passes.
        bank_trace keeps the reference's order (all forward frames, then all backward frames)."""
        pf = self._pass_setup(idx, True, lane=0)
        pb = self._pass_setup(idx, False, lane=1)
        cur = torch.cuda.current_stream(self.device)
        if self._lane_stream is None:
            self._lane_stream = torch.cuda.Stream(device=self.device)
        side = self._lane_stream
        side.wait_stream(cur)  # certain-memory copies, the interacted frame's memorize
        self._pass_streams = (cur, side)
        tf, tb = [], []
        nf, nb = len(pf[0].frames), len(pb[0].frames)
        for i in range(max(nf, nb)):
            if i < nf:
                self._pass_frame(*pf, pf[0].frames[i], key_k, idx, tf)
                if step_cb is not None:
                    step_cb()
            if i < nb:
                with torch.cuda.stream(side):
                    self._pass_frame(*pb, pb[0].frames[i], key_k, idx, tb)
                if step_cb is not None:
                    step_cb()
        cur.wait_stream(side)
        self._pass_streams = ()
        self.bank_trace.extend(tf + tb)

    def fuse_one_frame(self, tc, tr, ti, prev_mask, curr_mask, mk16, qk16):
        """inference_core.py:202-217.  `mk16` is the interacted frame's key in BANK layout
        [K,hw,128] when called from do_pass (or the reference layout [K,128,1,h,w]); `qk16` is the
        frame's QueryState (or the reference's k16 tensor)."""
        assert tc < ti < tr or tr < ti < tc
        nc = abs(tc - ti) / abs(tc - tr)
        nr = abs(tr - ti) / abs(tc - tr)
        if self._fuse_planes is None:
            self._fuse_planes = torch.zeros((self.k, 1, self.nh, self.nw), dtype=torch.float32, device=self.device)
        prob = self._fuse_planes
        im = self.get_image_buffered(ti)
        prev_mask = prev_mask.to(self.device).contiguous()
        for k in range(1, self.k + 1):
            if isinstance(qk16, QueryState):
                mk = mk16[k - 1] if mk16.dim() == 3 else mk16[k - 1].reshape(128, -1).t().contiguous()
                attn = self.prop_net.get_attention_resident(mk, qk16, self.pos_mask_diff[k:k + 1], self.neg_mask_diff[k:k + 1])
            else:
                attn = self.prop_net.get_attention(mk16[k - 1:k], self.pos_mask_diff[k:k + 1], self.neg_mask_diff[k:k + 1], qk16)
            self.fuse_net.forward_sigmoid_plane(im, prev_mask[k:k + 1].contiguous(), curr_mask[k:k + 1].contiguous(), attn,
                                                nc, nr, prob[k - 1, 0])
        return ops.aggregate_wbg(prob, keep_bg=True)

    # ------------------------------------------------------------------ interaction (:219-271)
    def interact(self, mask, idx, total_cb=None, step_cb=None):
        key_bank_k, key_v = self._begin_interaction(mask, idx, total_cb)
        if self._passes_can_overlap(idx):
            self._do_passes_overlapped(key_bank_k, key_v, idx, step_cb=step_cb)
        else:
            self.do_pass(key_bank_k, key_v, idx, True, step_cb=step_cb)
            self.do_pass(key_bank_k, key_v, idx, False, step_cb=step_cb)
        return self._finish_interaction()

    def _passes_can_overlap(self, idx) -> bool:
        """Both passes non-empty, graph replay on, the clip resident on the device (the host-clip staging slots
        of mem_profile >= 1 are recycled in issue order), and no pass bounded by another interaction (the fusion
        path shares FusionNet's workspace).  MIVOS_BIDIR=0 forces the sequential order."""
        if not self.overlap_passes or not self.use_graph or self.data_dev != self.device:
            return False
        if not (0 < idx < self.t - 1):
            return False
        return not any(ti != idx for ti in self.interacted)

    def _begin_interaction(self, mask, idx, total_cb=None):
        """inference_core.py:219-253: record the interaction, memorize the interacted frame as a certain
        memory, announce the number of frames the two passes will visit.  Returns the interacted
        frame's key in BANK layout [K,hw,128] and its value in the reference layout."""
        self.interacted.add(idx)
        mask = mask.to(self.device).float()
        mask, _ = pad_divide_by(mask, 16, mask.shape[-2:])
        mask = mask.contiguous()
        self.mask_diff = mask - self.prob[:, idx].to(self.device)  # uses the pre-interaction prob (:233)
        self.pos_mask_diff = self.mask_diff.clamp(0, 1)
        self.neg_mask_diff = (-self.mask_diff).clamp(0, 1)
        self.prob[:, idx] = mask

        K, hw = self.k, self.hw16
        key_bank_k = torch.empty((K, hw, 128), dtype=torch.float32, device=self.device)
        key_bank_v = torch.empty((K, hw, 512), dtype=torch.float32, device=self.device)
        self.prop_net.memorize_resident(self.get_image_buffered(idx), mask[1:], key_bank_k, key_bank_v, 0)
        key_k = key_bank_k.transpose(1, 2).reshape(K, 128, 1, self.kh, self.kw)  # reference layout (views)
        key_v = key_bank_v.transpose(1, 2).reshape(K, 512, 1, self.kh, self.kw)

        if self._certain_bank_k is None:
            self._certain_bank_k, self._certain_bank_v = key_bank_k, key_bank_v
            self.certain_mem_k, self.certain_mem_v = key_k, key_v
        else:  # :243-245
            self._certain_bank_k = torch.cat([self._certain_bank_k, key_bank_k], 1)
            self._certain_bank_v = torch.cat([self._certain_bank_v, key_bank_v], 1)
            self.certain_mem_k = torch.cat([self.certain_mem_k, key_k], 2)
            self.certain_mem_v = torch.cat([self.certain_mem_v, key_v], 2)

        if total_cb is not None:  # :247-253
            front_limit = min([ti for ti in self.interacted if ti > idx] + [self.t])
            back_limit = max([ti for ti in self.interacted if ti < idx] + [-1])
            total_num = front_limit - back_limit - 2
            if total_num > 0:
                total_cb(total_num)
        return key_bank_k, key_v

    def _finish_interaction(self):
        """inference_core.py:255-271: argmax over objects for every frame + unpad + u8 as one kernel, one
        asynchronous D2H into the pinned staging buffer, a fresh array for the caller."""
        ops.argmax_unpad(self.prob, self.pad, self.h, self.w, self.masks, self._masks_unpadded)
        self._masks_host.copy_(self._masks_unpadded, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        self.np_masks = self._masks_host.numpy().copy()
        return self.np_masks

    def reset(self):
        """Forget every interaction: the state of a freshly constructed InferenceCore over the same clip.
        The uploaded (or pinned) clip, the preallocated buffers and the shared network are kept; the
        query-feature cache is dropped, so the next interact() recomputes everything a new session
        would.  (Extension over the reference, which builds a new InferenceCore — and re-uploads the
        clip — per session: eval_interactive_davis.py:83.)"""
        cur = torch.cuda.current_stream(self.device)
        cur.wait_stream(self._qstream)  # nothing of the previous session is still in flight on the side stream
        self.prob.zero_()
        self.prob[0] = 1e-7  # :82
        self.masks.zero_()
        self._masks_unpadded.zero_()
        self.np_masks = np.zeros((self.t, self.h, self.w), dtype=np.uint8)
        self._query_pool.extend(self._query_chunks)
        self.query_buf, self._query_chunks, self._query_ready = {}, [], {}
        self.image_buf = {}
        self.interacted = set()
        self.certain_mem_k = self.certain_mem_v = None
        self._certain_bank_k = self._certain_bank_v = None
        self.bank_trace = []

    def update_mask_only(self, prob_mask, idx):
        """inference_core.py:273-292 — interaction only, no propagation."""
        prob_mask = prob_mask.to(self.device).float().contiguous()
        k1 = prob_mask.shape[0]
        nh, nw = prob_mask.shape[-2:]
        mp = torch.empty((1, 1, nh, nw), dtype=torch.uint8, device=self.device)
        mo = torch.empty((1, self.h, self.w), dtype=torch.uint8, device=self.device)
        ops.argmax_unpad(prob_mask.reshape(k1, 1, 1, nh, nw), self.pad, self.h, self.w, mp, mo)
        self.masks[idx] = mp[0]
        self.np_masks[idx] = mo[0].cpu().numpy()
        return self.np_masks
