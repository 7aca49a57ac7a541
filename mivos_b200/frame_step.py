"""The per-frame step of the propagation loop, for one clip (``InferenceCore``) or for C clips that advance
together (``LockstepSession``): a single clip is the case C = 1."""
from __future__ import annotations

import weakref
from typing import Optional, Sequence

import torch

from . import _lib, ops
from ._lib import MivosError
from .host_results import HostResults


class FrameStep:
    """One propagated frame of C clips (memory read -> decoder -> aggregate [-> memorize trunk -> bank write]) as a
    captured CUDA graph.  The C*K object maps go through every convolution as ONE batch (C times the row tiles per
    launch); the operators whose operands differ per clip take the C clips as groups of one launch
    (engine.PropagationEngine.segment / encode_memory).  Everything that changes from frame to frame lives in device
    memory the graph reads: each clip's frame and query-side features (from its batched query pass,
    InferenceCore.get_query_kv_buffered) are staged into `frames[c]` / `batch`, the live bank size and the bank slot of
    the memorize are the int32 scalars `dyn` (identical for all clips: they execute one plan), results land in
    `prob[c]`.  One graph with and one without the memorize serve every frame of every pass while the bank grows, so
    the kernel launches of a frame cost one graph launch on the host.  Instances (with their bank buffers) are
    cached on the network's engine and shared by successive sessions — the reference also shares the networks between
    sessions (eval_interactive_davis.py:83)."""

    def __init__(self, net, C: int, K: int, nh: int, nw: int, cap_frames: int, lane: int = 0, ragged: bool = False,
                 maps: Optional[int] = None):
        eng = net.engine()
        dev = eng.device
        # the step is cached on the network's engine: a strong reference back would be a cycle that keeps a dropped
        # network's workspaces, banks and graphs in device memory until the garbage collector happens to run
        self.net = weakref.proxy(net)
        self.C, self.K, self.nh, self.nw, self.lane = C, K, nh, nw, lane
        self.hw = (nh // 16) * (nw // 16)
        self.cap_frames = cap_frames
        # mixed object counts (ragged, `maps` = the clips' total object count): bank rows, result planes and
        # destination pointers are sized for the maps, not for C*K; the planes are PACKED [maps + C,1,nh,nw] (each
        # clip's background plane, then its objects) and a device table `first` [C+1] says which clip owns which
        self.maps = maps
        N, P = (C * K, C * (K + 1)) if maps is None else (maps, maps + C)
        self.frames = torch.zeros((C, 3, nh, nw), dtype=torch.float32, device=dev)
        self.prob = torch.zeros(((C, K + 1) if maps is None else (P,)) + (1, nh, nw), dtype=torch.float32, device=dev)
        self.dyn = torch.zeros(4, dtype=torch.int32, device=dev)
        states, self.batch = eng.new_query_states(nh, nw, C)
        # one clip keeps the single-clip operands: [hw,128] query keys (read without query sets), [K+1,1,H,W] planes
        if maps is None:
            self.q, self.out = (states[0], self.prob[0]) if C == 1 else (self.batch, self.prob)
            self.masks = self.out.narrow(-4, 1, K)  # the object planes the memorize reads
        self.bank_k = torch.empty((N, cap_frames * self.hw, 128), dtype=torch.float32, device=dev)
        self.bank_v = torch.empty((N, cap_frames * self.hw, 512), dtype=torch.float32, device=dev)
        self.graphs = {}
        self.kernels = {}  # kernels per replay, for mivos_launch_count accounting
        # False: eager launches even when the caller asks for graph replay (bench.py's per-launch brackets)
        self.use_graph = True
        # Device pointer table of the step (mivos_copy_segments): the graph STAGES each clip's operands itself — frame,
        # cached query features kv / qk / s8 / s4: source pointers in dynp[:5C] — and DELIVERS its K+1 result planes to
        # InferenceCore.prob[:, ti] (destination pointers in dynp[5C:]); per frame the host writes the table and the two
        # bank counters with ONE small launch (mivos_store_words) and replays the graph: no eager copy.
        b = self.batch
        staged = [t for c in range(C) for t in (self.frames[c], b.kv[c], b.qk[c], b.s8[c], b.s4[c])]
        i64 = lambda v: torch.tensor(v, dtype=torch.int64, device=dev)  # noqa: E731
        self.g_fixed = i64([t.data_ptr() for t in staged])
        self.g_bytes_host = [t.numel() * t.element_size() for t in staged]
        self.g_bytes = i64(self.g_bytes_host)
        planes = self.prob.view(P, 1, nh, nw)
        self.s_fixed = i64([planes[j].data_ptr() for j in range(P)])
        self.plane_bytes = nh * nw * 4
        self.s_bytes = i64([self.plane_bytes] * P)
        # ragged (clips with their own pass plans, LockstepSession): C more words of the table hold one live slot
        # count and one memorize frame per clip, as int32 `counts` [2C] = (slots of clips 0..C-1, frames of clips
        # 0..C-1), written with the pointers; a tick of the first n of the C clips runs over their leading rows
        # (mixed: (C + 2) // 2 more words hold the int32 group table `first` [C+1] of the tick's clip order)
        self.ragged = ragged or maps is not None
        words = 5 * C + P
        # host results (InferenceCore(result_dev="cpu")): one mivos_deliver_planes record per clip follows, written
        # only in the ticks that have such a clip; a tick of device-result clips writes and launches what it always did
        self.d_off = words + (C if self.ragged else 0) + ((C + 2) // 2 if maps is not None else 0)
        self.dynp = torch.zeros(self.d_off + C * ops.DELIVER_WORDS, dtype=torch.int64, device=dev)
        self.counts = self.dynp[words:words + C].view(torch.int32) if self.ragged else None
        self.first = self.dynp[words + C:].view(torch.int32)[:C + 1] if maps is not None else None
        self.records = self.dynp[self.d_off:]

    @staticmethod
    def get(net, C: int, K: int, nh: int, nw: int, need_frames: int, lane: int = 0, ragged: bool = False,
            maps: Optional[int] = None) -> "FrameStep":
        """The cached step for these shapes.  Single clips are kept in the engine's `_frame_steps` (4 entries),
        lock-step groups, whose C*K banks are C times larger, in `_lock_steps` (2 entries); least recently used
        first out."""
        name, bound = ("_frame_steps", 4) if C == 1 else ("_lock_steps", 2)
        cache = net.engine().__dict__.setdefault(name, {})
        cap = (need_frames + 15) // 16 * 16
        key = (C, K, nh, nw, cap, lane) + (("ragged",) if ragged else ()) + (("maps", maps) if maps is not None else ())
        step = cache.pop(key, None)
        if step is None:
            step = FrameStep(net, C, K, nh, nw, cap, lane, ragged, maps)
            while len(cache) >= bound:  # dict order = use order
                cache.pop(next(iter(cache)))
        cache[key] = step  # (re)insert as most recently used
        return step

    def _body(self, memorize: bool, host: bool = False):
        eng, C, K = self.net.engine(), self.C, self.K
        with eng.lane(self.lane):
            ops.copy_segments(self.g_fixed, self.dynp, self.g_bytes, 5 * C, True, max(self.g_bytes_host))
            eng.segment(self.bank_k, self.bank_v, self.cap_frames * self.hw, self.q, K, C, prob_out=self.out,
                        dyn_slots=self.dyn[0:1])
            if memorize:
                # the C*K object banks are contiguous and share the frame slot: one bank write per object chunk
                eng.memorize_into(self.frames, self.masks, self.bank_k, self.bank_v, self.cap_frames - 1,
                                  dyn_t=self.dyn[1:2])
            ops.copy_segments(self.s_fixed, self.dynp[5 * C:], self.s_bytes, C * (K + 1), False, self.plane_bytes)
            if host:
                ops.deliver_planes(self.prob, self.records, C, self.nh, self.nw)

    def _body_ragged(self, n: int, n_mem: int, host: bool = False):
        """A tick of the first n clips, the first n_mem of them memorizing: the same operators as _body over the
        leading n (n_mem) clips, the reads and the bank write in their per-set forms (counts per clip)."""
        eng, C, K = self.net.engine(), self.C, self.K
        with eng.lane(self.lane):
            ws = eng.ws
            ops.copy_segments(self.g_fixed, self.dynp, self.g_bytes, 5 * n, True, max(self.g_bytes_host))
            with ws.prefix_of(n * K, C * K):
                eng.segment(self.bank_k[:n * K], self.bank_v[:n * K], self.cap_frames * self.hw, self.batch.first(n), K,
                            n, prob_out=self.prob[0] if n == 1 else self.prob[:n], dyn_slots=self.counts[:n],
                            dyn_sets=True)
            if n_mem:
                with ws.prefix_of(n_mem * K, C * K):
                    eng.memorize_into(self.frames[:n_mem], self.prob[:n_mem].narrow(-4, 1, K), self.bank_k[:n_mem * K],
                                      self.bank_v[:n_mem * K], self.cap_frames - 1, dyn_t=self.counts[C:C + n_mem],
                                      dyn_sets=True)
            ops.copy_segments(self.s_fixed, self.dynp[5 * C:], self.s_bytes, n * (K + 1), False, self.plane_bytes)
            if host:
                ops.deliver_planes(self.prob, self.records, n, self.nh, self.nw)

    def _body_mixed(self, n: int, n_mem: int, mn: int, mm: int, host: bool = False):
        """A tick of the first n clips of a mixed step, the first n_mem memorizing: _body_ragged over object groups.
        The clips' mn (mm) object maps are the leading bank rows and planes; the reads, the decoder's per-clip
        operators, the aggregation, the memorize stem and the bank write take the group table `first`."""
        eng, C, N = self.net.engine(), self.C, self.maps
        with eng.lane(self.lane):
            ws = eng.ws
            ops.copy_segments(self.g_fixed, self.dynp, self.g_bytes, 5 * n, True, max(self.g_bytes_host))
            with ws.prefix_of(mn, N):
                eng.segment(self.bank_k[:mn], self.bank_v[:mn], self.cap_frames * self.hw, self.batch.first(n), mn, n,
                            prob_out=self.prob[:mn + n], dyn_slots=self.counts[:n], first=self.first[:n + 1])
            if n_mem:
                with ws.prefix_of(mm, N):
                    eng.memorize_into(self.frames[:n_mem], self.prob[:mm + n_mem], self.bank_k[:mm], self.bank_v[:mm],
                                      self.cap_frames - 1, dyn_t=self.counts[C:C + n_mem], first=self.first[:n_mem + 1])
            ops.copy_segments(self.s_fixed, self.dynp[5 * C:], self.s_bytes, mn + n, False, self.plane_bytes)
            if host:
                ops.deliver_planes(self.prob, self.records, n, self.nh, self.nw)

    def run_ragged(self, frames: Sequence[Optional[torch.Tensor]], cached, visible: Sequence[int],
                   m_front: Sequence[int], n_mem: int, prob_dsts, ti: Sequence[int], graph: bool = True,
                   ks: Optional[Sequence[int]] = None) -> torch.Tensor:
        """One tick of the first n = len(cached) clips of a ragged step, each at its own frame: clip c reads
        visible[c] bank frames and (c < n_mem) memorizes into frame m_front[c]; frames[c] / cached[c] / ti[c] as in
        run, prob_dsts[c] clip c's destination volume, its HostResults, or None (fused frame: the planes stay in
        self.prob[c]).  The
        pointers and the per-clip counters are written with one store; one captured graph per (n, n_mem)."""
        assert self.ragged
        n, C, K = len(cached), self.C, self.K
        assert 1 <= n <= C and 0 <= n_mem <= n
        mixed = self.maps is not None
        if mixed:  # object counts of the clips in this tick's order, then of the rest of the C clips
            assert ks is not None and len(ks) == C and sum(ks) == self.maps
            first = [0]
            for k in ks:
                first.append(first[-1] + k)
        srcs, dsts, slots, mem_t, recs = [], [], [], [], []
        for c in range(C):
            if c < n:
                assert visible[c] <= self.cap_frames and m_front[c] < self.cap_frames
                if visible[c] * self.hw < self.net.min_live_slots:  # same rule as mivos_memory_read and torch.topk
                    raise MivosError(f"memory_read: clip {c}: {visible[c] * self.hw} live bank slots < top_k "
                                     f"{self.net.top_k}")
                q = cached[c]
                srcs += [frames[c].data_ptr() if c < n_mem else 0, q.kv.data_ptr(), q.qk.data_ptr(), q.s8.data_ptr(),
                         q.s4.data_ptr()]
                d = prob_dsts[c]
                kc = ks[c] if mixed else K
                if isinstance(d, HostResults):  # the clip's planes: packed (background, then its objects) or row c
                    recs += d.record(ti[c], first[c] + c if mixed else c * (K + 1))
                    d = None
                else:
                    recs += [0] * ops.DELIVER_WORDS
                dsts += [d[j, ti[c]].data_ptr() for j in range(kc + 1)] if d is not None else [0] * (kc + 1)
                slots.append(visible[c] * self.hw)
                mem_t.append(m_front[c] if c < n_mem else 0)
            else:
                srcs += [0] * 5
                dsts += [0] * ((ks[c] if mixed else K) + 1)
                slots.append(0)
                mem_t.append(0)
        i32 = slots + mem_t
        if mixed:
            i32 += first + [0] * ((C + 2) // 2 * 2 - (C + 1))
        packed = [(i32[2 * i] & 0xFFFFFFFF) | ((i32[2 * i + 1] & 0xFFFFFFFF) << 32) for i in range(len(i32) // 2)]
        packed = [w - (1 << 64) if w >= 1 << 63 else w for w in packed]
        host = any(recs)
        ops.store_words(self.dynp, srcs + dsts + packed + (recs if host else []))
        # a mixed step's graphs are keyed by the map counts of the two prefixes too (the table itself is device data),
        # and every step's by the delivery kind
        args = (n, n_mem, first[n], first[n_mem]) if mixed else (n, n_mem)
        body = self._body_mixed if mixed else self._body_ragged
        if not (graph and self.use_graph):
            body(*args, host=host)
            return self.prob
        lib = _lib.load()
        key = args + ("host",) if host else args
        g = self.graphs.get(key)
        if g is None:
            n0 = lib.mivos_launch_count()
            body(*args, host=host)
            self.kernels[key] = lib.mivos_launch_count() - n0
            torch.cuda.current_stream().synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                body(*args, host=host)
            lib.mivos_add_launch_count(-self.kernels[key])
            self.graphs[key] = g
            # the eager run above was this tick: a replay would run it twice, and a prefix first appears mid-pass,
            # where a clip's read may see the temporary bank frame its memorize has just overwritten
            return self.prob
        g.replay()
        lib.mivos_add_launch_count(self.kernels[key])
        return self.prob

    def run(self, frames: Sequence[Optional[torch.Tensor]], cached, visible: int, m_front: int, memorize: bool,
            prob_dsts=None, ti: int = 0, graph: bool = True) -> torch.Tensor:
        """`frames[c]` [1,3,nh,nw] (device; read when memorizing) and `cached[c]` the QueryState of clip c's frame;
        `prob_dsts[c]` [(K+1),T,1,nh,nw]: the step writes clip c's result planes to prob_dsts[c][:, ti] itself (None:
        they are only left in self.prob[c], e.g. for fuse_one_frame); a HostResults (host volumes) gets them, with the
        frame's labels, from one mivos_deliver_planes launch for all such clips.  `graph`: replay the captured graph (the
        calling session's use_graph), else launch eagerly.  Returns self.prob [C,K+1,1,nh,nw]."""
        assert visible <= self.cap_frames and m_front < self.cap_frames
        if visible * self.hw < self.net.min_live_slots:  # same rule as mivos_memory_read and torch.topk
            raise MivosError(f"memory_read: {visible * self.hw} live bank slots < top_k {self.net.top_k}")
        srcs, dsts, recs = [], [], []
        for c in range(self.C):
            q = cached[c]
            srcs += [frames[c].data_ptr() if memorize else 0, q.kv.data_ptr(), q.qk.data_ptr(), q.s8.data_ptr(),
                     q.s4.data_ptr()]
            d = prob_dsts[c] if prob_dsts is not None else None
            if isinstance(d, HostResults):
                recs += d.record(ti, c * (self.K + 1))
                d = None
            else:
                recs += [0] * ops.DELIVER_WORDS
            dsts += [d[j, ti].data_ptr() for j in range(self.K + 1)] if d is not None else [0] * (self.K + 1)
        host = any(recs)
        ops.store_words(self.dynp, srcs + dsts + (recs if host else []), self.dyn, (visible * self.hw, m_front))
        if not (graph and self.use_graph):
            self._body(memorize, host)
            return self.prob
        lib = _lib.load()
        key = (memorize, "host") if host else memorize
        g = self.graphs.get(key)
        if g is None:
            # first use: run eagerly once (allocates every workspace, sets kernel attributes), then capture
            n0 = lib.mivos_launch_count()
            self._body(memorize, host)
            self.kernels[key] = lib.mivos_launch_count() - n0
            torch.cuda.current_stream().synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._body(memorize, host)
            lib.mivos_add_launch_count(-self.kernels[key])  # capture issued no work
            self.graphs[key] = g
        g.replay()
        lib.mivos_add_launch_count(self.kernels[key])
        return self.prob
