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
from ._lib import MivosError
from .engine import QueryState, object_chunks
from .frame_step import FrameStep
from .host_results import HostResults
from .tensor_util import pad_divide_by


class InferenceCore:
    def __init__(self, prop_net, fuse_net, images, num_objects, mem_profile=0, mem_freq=5, device="cuda:0",
                 result_dev=None):
        """`result_dev`: None keeps prob / masks on the device, for every mem_profile; "cpu" keeps them in
        page-locked host memory (host_results.HostResults), as the reference's result_dev = 'cpu' does: the
        device footprint then does not grow with the clip's length, and the results are the same bits."""
        if result_dev is not None and str(result_dev) != "cpu":  # "cpu" or torch.device("cpu")
            raise MivosError(f"InferenceCore: result_dev must be None or 'cpu', got {result_dev!r}")
        self.device = torch.device(device)
        _lib.require_cuda_device(self.device, "mivos_b200.InferenceCore")
        self.prop_net = prop_net.to(self.device, non_blocking=True)
        if fuse_net is not None:
            self.fuse_net = fuse_net.to(self.device, non_blocking=True)
        self.mem_profile = mem_profile
        self.mem_freq = mem_freq

        # Same buffer policy table as the reference (:44-63), except for result_dev: results live on the device
        # unless the caller asks for host results (a 480p prob volume is 1.66 MB per frame per object); the
        # query-feature cache honours q_buf_size, image staging honours data_dev / i_buf_size.
        if mem_profile == 0:
            self.data_dev, self.q_buf_size, self.i_buf_size = self.device, 105, -1
        elif mem_profile == 1:
            self.data_dev, self.q_buf_size, self.i_buf_size = torch.device("cpu"), 105, 105
        elif mem_profile == 2:
            self.data_dev, self.q_buf_size, self.i_buf_size = torch.device("cpu"), 3, 3
        else:
            self.data_dev, self.q_buf_size, self.i_buf_size = torch.device("cpu"), 1, 1
        self.result_dev = self.device if result_dev is None else torch.device("cpu")

        t = images.shape[1]
        h, w = images.shape[-2:]
        ops.check_objects(num_objects, "InferenceCore")
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

        self.np_masks = np.zeros((t, h, w), dtype=np.uint8)
        # host results: prob, masks (:77-82) and the label maps the deliveries keep in page-locked host volumes
        self._host = None if result_dev is None else HostResults(self.k + 1, t, nh, nw, h, w, self.pad, self.device)
        if self._host is None:
            self.masks = torch.zeros((t, 1, nh, nw), dtype=torch.uint8, device=self.result_dev)  # :77
            # result masks cross PCIe into ONE pinned staging buffer (async D2H at link rate instead of a
            # pageable copy); interact() hands the caller a fresh array copied from it, as the reference's
            # `.cpu().numpy()` does (:269)
            self._masks_host = torch.zeros((t, h, w), dtype=torch.uint8).pin_memory()
            self.prob = torch.zeros((self.k + 1, t, 1, nh, nw), dtype=torch.float32, device=self.result_dev)  # :81
            self.prob[0] = 1e-7  # :82
        else:
            self.masks, self.prob, self._masks_host = self._host.masks, self._host.prob, None

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
        self._masks_unpadded = None if self._host else torch.zeros((t, h, w), dtype=torch.uint8, device=self.device)
        self._fuse_planes = None
        self.bank_trace = []  # (frame, visible bank frames) per propagated frame, for plumbing tests
        # CUDA-graph replay of the per-frame step (MIVOS_GRAPH=0: the step's launches are issued eagerly)
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
    def do_pass(self, key_k, key_v, idx, forward=True, step_cb=None):
        return run_pass([self], [key_k], idx, forward, step_cb)

    def _do_passes_overlapped(self, key_k, key_v, idx, step_cb=None):
        """The forward and the backward pass of one interaction are independent until the argmax
        (inference_core.py:255-256): they run here as two LANES — own frame-step graphs, bank, workspace
        (engine.lane(1)) and CUDA stream — issued frame by frame in alternation, so the kernels of one
        pass fill the SMs the other's latency-bound chain leaves idle.  Each pass executes exactly the
        launches of do_pass in the same order: results are bit-identical to the sequential passes.
        bank_trace keeps the reference's order (all forward frames, then all backward frames)."""
        pf = _pass_setup([self], idx, True, lane=0)
        pb = _pass_setup([self], idx, False, lane=1)
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
                _pass_frame([self], *pf, pf[0].frames[i], [key_k], idx, [tf])
                if step_cb is not None:
                    step_cb()
            if i < nb:
                with torch.cuda.stream(side):
                    _pass_frame([self], *pb, pb[0].frames[i], [key_k], idx, [tb])
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
        return ops.aggregate_any(prob, keep_bg=True)

    # ------------------------------------------------------------------ result frames
    def _results(self):
        """Where a frame step delivers this clip's result planes: its prob volume or its host volumes."""
        return self.prob if self._host is None else self._host

    def _frame(self, ti):
        """prob[:, ti] on the device."""
        return self.prob[:, ti] if self._host is None else self._host.load(ti)

    def _set_frame(self, ti, planes):
        """prob[:, ti] = planes [(K+1),1,nh,nw] (device); host results get the frame's labels with them."""
        if self._host is None:
            self.prob[:, ti] = planes
        else:
            self._host.store(planes, ti)

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
        path shares FusionNet's workspace), and no more objects than one chunk (object_chunks): a second lane would
        hold a second bank, 34 GB at 255 objects over 101 480p frames.  MIVOS_BIDIR=0 forces the sequential order."""
        if len(object_chunks(self.k)) > 1:
            return False
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
        self._set_frame(idx, mask)

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
        asynchronous D2H into the pinned staging buffer, a fresh array for the caller.  Host results: the
        deliveries have kept the label maps at argmax(prob) of every frame, so after one synchronisation masks and
        the returned array are host copies of them."""
        if self._host is not None:
            torch.cuda.current_stream(self.device).synchronize()
            self.masks.copy_(self._host.labels)
            self.np_masks = self._host.labels_unpadded.numpy().copy()
            return self.np_masks
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
        if self._host is not None:
            cur.synchronize()  # no delivery is still writing the host volumes
            self._host.fill()
        else:
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


# ---------------------------------------------------------------------- the pass loop, for one clip or C lock-step clips
def run_pass(cores, keys, idx, forward, step_cb=None):
    """One pass (:122-200) of every clip of `cores` (InferenceCore objects that share one pass plan: one clip, or
    the clips of a LockstepSession) from the interacted frame `idx`; keys[c]: clip c's interacted key in BANK
    layout.  step_cb() once per frame of the pass.  Returns the frame that bounds the pass."""
    plan, step = _pass_setup(cores, idx, forward)
    for fp in plan.frames:
        _pass_frame(cores, plan, step, fp, keys, idx, [core.bank_trace for core in cores])
        if step_cb is not None:
            step_cb()
    return plan.closest_ti


def _pass_setup(cores, idx, forward, lane: int = 0):
    """Plan of one pass (:128-141), the frame step that serves it (lane 0 or 1) and every clip's certain memories
    copied into its banks (:146-151)."""
    c0 = cores[0]
    K, hw = c0.k, c0.hw16
    num_certain = c0._certain_bank_k.shape[1] // hw
    # the bank bookkeeping of the pass (:128-141, :166-186) is host arithmetic: schedule.plan_pass
    plan = schedule.plan_pass(c0.t, c0.interacted, idx, forward, c0.mem_freq, num_certain)
    if not plan.frames:
        return plan, None
    # bank sized for the longest pass of this clip plus a fixed interaction budget, so the bank
    # pointers (and with them the captured graphs) stay valid across passes and sessions
    step = FrameStep.get(c0.prop_net, len(cores), K, c0.nh, c0.nw,
                         schedule.bank_capacity_frames(c0.t, c0.mem_freq, num_certain, plan.total_m), lane)
    for c, core in enumerate(cores):
        step.bank_k[c * K:(c + 1) * K, :num_certain * hw].copy_(core._certain_bank_k)
        step.bank_v[c * K:(c + 1) * K, :num_certain * hw].copy_(core._certain_bank_v)
    return plan, step


def _pass_frame(cores, plan, step, fp, keys, idx, traces):
    """One propagated frame of a pass (:165-194) for every clip, on the current stream.  The first core's use_graph
    decides between graph replay and eager launches."""
    ti = fp.ti
    cached = [core.get_query_kv_buffered(ti, plan.step, plan.closest_ti) for core in cores]  # :172
    # the step stages its operands and (unless the frame is fused) writes every clip's prob[:, ti] itself  # :173-179, :194
    frames = [core.get_image_buffered(ti) if fp.memorize else None for core in cores]
    prob = step.run(frames, cached, fp.visible, fp.m_front, fp.memorize,
                    prob_dsts=None if plan.fuse else [core._results() for core in cores], ti=ti, graph=cores[0].use_graph)
    for c, core in enumerate(cores):
        traces[c].append((ti, fp.visible))
        if plan.fuse:  # :190-194
            core._set_frame(ti, core.fuse_one_frame(plan.closest_ti, idx, ti, core._frame(ti), prob[c], keys[c], cached[c]))
