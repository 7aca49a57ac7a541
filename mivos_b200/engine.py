"""Layer graphs of the propagation path, executed as sequences of C-ABI kernel launches on HALO
buffers (include/mivos_b200.h).  This is the host-side scheduler of the hot path: weights are
packed once (BatchNorm folded, K-major, TF32-rounded), activations stay resident in HBM in the
layout the implicit-GEMM kernel consumes, and nothing is allocated per frame.

Reference semantics followed (paths relative to the reference root):
  * ResNet-50 trunks to layer3, with / without mask channels — model/propagation/modules.py:38-89,
    mod_resnet.py:76-150
  * key/value projections — modules.py:107-114
  * memory read + decoder + sigmoid — prop_net.py:14-31, 81-108, 170-181
  * FusionNet — model/fusion_net.py:32-50
"""
from __future__ import annotations

import contextlib
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

from . import arch, ops
from ._lib import MivosError
from .ops import PackedConv

BN_EPS = 1e-5
CHUNK_OBJECTS = 16  # most object maps one memorize / decoder batch takes


def object_chunks(K: int):
    """(first object, count) of the object chunks a clip of K objects runs its memorize and decoder in: one chunk up
    to CHUNK_OBJECTS, else ceil(K / CHUNK_OBJECTS) chunks of near-equal size (the larger ones first), so that every
    convolution keeps a batch shape of at most CHUNK_OBJECTS maps and its workspace stays at that size."""
    if K <= CHUNK_OBJECTS:
        return [(0, K)]
    m = -(-K // CHUNK_OBJECTS)
    q, r = divmod(K, m)
    chunks, k0 = [], 0
    for i in range(m):
        n = q + (1 if i < r else 0)
        chunks.append((k0, n))
        k0 += n
    return chunks


class Workspace:
    """Named, shape-keyed device buffers.  HALO buffers are zeroed once at creation; kernels never
    write the border, so reuse across layers and frames keeps the zero-padding invariant."""

    def __init__(self, device, dtype=torch.float32):
        self.device = device
        self.dtype = dtype  # element type of activation maps (fp32 for the TF32 path, or fp16)
        self._bufs: Dict[tuple, torch.Tensor] = {}
        self._prefix = None  # (n, full) inside prefix_of()

    @contextlib.contextmanager
    def prefix_of(self, n: int, full: int):
        """Inside the block, a buffer of n maps (a HALO map of n images, a matrix of n images' rows) is the leading
        part of the buffer of `full` maps: a batch of the first n of `full` lock-step clips allocates nothing the
        full batch does not.  HALO maps and gathered matrices are image-major, so the prefix is contiguous."""
        prev, self._prefix = self._prefix, (n, full)
        try:
            yield
        finally:
            self._prefix = prev

    def full(self, n: int) -> int:
        """The map count a buffer of n maps is allocated for (see prefix_of)."""
        return self._prefix[1] if self._prefix is not None and n == self._prefix[0] else n

    def halo(self, tag: str, n: int, h: int, w: int, c: int, dtype=None) -> torch.Tensor:
        dtype = dtype or self.dtype
        if self._prefix is not None and n == self._prefix[0] and n != self._prefix[1]:
            return self.halo(tag, self._prefix[1], h, w, c, dtype)[:n]
        key = ("halo", tag, n, h, w, c, dtype)
        buf = self._bufs.get(key)
        if buf is None:
            buf = ops.halo_zeros(n, h, w, c, self.device, dtype)
            self._bufs[key] = buf
        return buf

    def mat(self, tag: str, rows: int, cols: int, dtype=None) -> torch.Tensor:
        dtype = dtype or self.dtype
        if self._prefix is not None and self._prefix[0] != self._prefix[1] and rows % self._prefix[0] == 0:
            full = rows // self._prefix[0] * self._prefix[1]
            prev, self._prefix = self._prefix, None  # the full-size lookup itself
            try:
                return self.mat(tag, full, cols, dtype)[:rows]
            finally:
                self._prefix = prev
        key = ("mat", tag, rows, cols, dtype)
        buf = self._bufs.get(key)
        if buf is None:
            buf = torch.zeros((rows, cols), dtype=dtype, device=self.device)
            self._bufs[key] = buf
        return buf

    def splitk(self) -> torch.Tensor:
        """Zero-initialised split-K scratch of mivos_conv_gemm, private to this workspace (= to the
        stream its launches are issued on)."""
        buf = self._bufs.get(("splitk",))
        if buf is None:
            buf = ops.split_k_workspace(self.device)
            self._bufs[("splitk",)] = buf
        return buf

    def raw(self, tag: str, nbytes: int) -> torch.Tensor:
        """Scratch bytes, in power-of-two size classes.  A buffer is never replaced or freed once handed
        out: captured CUDA graphs keep raw pointers into it (a grow-and-replace policy would leave the
        graphs of a smaller configuration pointing at freed memory)."""
        size = 1 << max(20, (max(nbytes, 1) - 1).bit_length())
        key = ("raw", tag, size)
        buf = self._bufs.get(key)
        if buf is None:
            buf = torch.empty(size, dtype=torch.uint8, device=self.device)
            self._bufs[key] = buf
        return buf

    def bytes(self) -> int:
        return sum(b.numel() * b.element_size() for b in self._bufs.values())


@dataclass
class QueryState:
    """Per-frame query-side features kept resident (HALO layout) — everything of a propagated
    frame that depends on the frame alone and not on the propagation state:
      kv [1,H/16,W/16,640] = key(128) | value(512)   (kv_q_f16, prop_net.py:166)
      qk [hw,128]          pixel-major copy of the key channels for the memory read
      s8 [1,H/8,W/8,512], s4 [1,H/4,W/4,256]  outputs of the decoder's SKIP paths
          skip_conv2(skip_conv1(f8 | f4)) (modules.py:101): 184 of the decoder's 321 GFLOP.  They
          are a function of the frame only, so they are produced by the (batched) query pass and
          the per-frame decoder starts at the bilinear add.
    f16/f8/f4 are only kept when the reference-layout API needs to return them."""

    kv: torch.Tensor
    qk: torch.Tensor
    s8: torch.Tensor
    s4: torch.Tensor
    h: int
    w: int
    f16: Optional[torch.Tensor] = None
    f8: Optional[torch.Tensor] = None
    f4: Optional[torch.Tensor] = None

    def first(self, n: int) -> "QueryState":
        """The first n frames of a batched state (views, no copy)."""
        cut = lambda t: None if t is None else t[:n]  # noqa: E731
        return QueryState(kv=self.kv[:n], qk=self.qk[:n], s8=self.s8[:n], s4=self.s4[:n], h=self.h, w=self.w,
                          f16=cut(self.f16), f8=cut(self.f8), f4=cut(self.f4))


def _cg(ws: "Workspace", *args, **kw):
    """mivos_conv_gemm with the workspace's split-K scratch attached."""
    return ops.conv_gemm(*args, splitk_ws=ws.splitk(), **kw)


def _bn_of(sd, name):
    return (sd[name + ".weight"], sd[name + ".bias"], sd[name + ".running_mean"], sd[name + ".running_var"], BN_EPS)


def act_dtype_from_env(default: Optional[str] = None) -> torch.dtype:
    """Element type of the convolution operands / activation maps when the network constructor was not
    given one.  Order: MIVOS_ACT_DTYPE = tf32 | fp16; else the caller's precision context, like the
    reference's nn.Modules: fp16 under ``torch.autocast`` (the GUI wraps every call in
    ``torch.cuda.amp.autocast``, interactive_gui.py:990), TF32 otherwise (the DAVIS evaluation and every
    other caller run the reference in fp32: eval_interactive_davis.py, davis_processor.py).
    tf32: fp32 storage, kind::tf32 MMAs with round-to-nearest operands — the fp32-comparable path.
    fp16: fp16 storage (half the bytes through TMA / L2 / HBM), kind::f16 MMAs.  Accumulation, bias,
    key/value bank, memory read, logits and probabilities are fp32 either way."""
    import os
    v = os.environ.get("MIVOS_ACT_DTYPE", default or "").lower()
    if not v:
        return torch.float16 if torch.is_autocast_enabled() else torch.float32
    if v in ("tf32", "fp32", "float32"):
        return torch.float32
    if v in ("fp16", "f16", "half", "float16"):
        return torch.float16
    raise ValueError(f"MIVOS_ACT_DTYPE={v!r}: expected tf32 or fp16")


class _ResNetTrunk:
    """ResNet-50 bottleneck stages on HALO maps, shared by the propagation encoders and the S2M
    backbone.  Needs ``self.pc`` (name -> PackedConv)."""

    pc: Dict[str, PackedConv]

    def _bottleneck(self, p, x, n, h, w, cin, planes, stride, has_ds, out, ws, dilation=1):
        """mod_resnet.py:76-112 / s2m_resnet.py:27-66.  stride 2: the 3x3 (and the 1x1 downsample) read a
        strided gather; dilation > 1 (stride 1): the 3x3 reads a dilated gather; otherwise the HALO
        map directly."""
        pc = self.pc
        ho, wo = h // stride, w // stride
        t1 = ws.halo("t1", n, h, w, planes)
        _cg(ws, x, pc[f"{p}.conv1"], n, h, w, t1, relu=True, round_tf32=True)
        t2 = ws.halo("t2", n, ho, wo, planes)
        if stride == 1 and dilation == 1:
            _cg(ws, t1, pc[f"{p}.conv2"], n, h, w, t2, relu=True, round_tf32=True)
        elif stride == 1:
            gd = ws.mat("gd", n * (h + 2) * (w + 2), 9 * planes)
            ops.gather_dilated(t1, n, h, w, planes, dilation, gd)
            _cg(ws, gd, pc[f"{p}.conv2"], n, h, w, t2, relu=True, round_tf32=True)
        else:
            assert dilation == 1
            g3 = ws.mat("g3", n * (ho + 2) * (wo + 2), 9 * planes)
            ops.gather_s2(t1, n, h, w, planes, 3, g3)
            _cg(ws, g3, pc[f"{p}.conv2"], n, ho, wo, t2, relu=True, round_tf32=True)
        res = x
        if has_ds:
            res = ws.halo("ds", n, ho, wo, 4 * planes)
            if stride == 1:
                _cg(ws, x, pc[f"{p}.downsample.0"], n, h, w, res)
            else:
                g1 = ws.mat("g1", n * (ho + 2) * (wo + 2), cin)
                ops.gather_s2(x, n, h, w, cin, 1, g1)
                _cg(ws, g1, pc[f"{p}.downsample.0"], n, ho, wo, res)
        _cg(ws, t2, pc[f"{p}.conv3"], n, ho, wo, out, relu=True, residual=res, round_tf32=True)
        return out

    def _trunk(self, prefix, lnames, stem_mat, n, H, W, keep: Dict[int, torch.Tensor], ws: "Workspace",
               planes_t=arch.TRUNK_PLANES, blocks_t=arch.TRUNK_BLOCKS, strides_t=arch.TRUNK_STRIDES, dilation_t=None):
        """stem_mat: gathered 7x7/2 windows [n*(H/2+2)*(W/2+2), kpad].  `keep[i]` is the caller's
        buffer for the output of layer i (0: 1/4, 1: 1/8, 2: 1/16, ...); other outputs ping-pong.
        dilation_t[i] = (dilation of the first block, dilation of the others) of layer i."""
        pc = self.pc
        h2, w2 = H // 2, W // 2
        s1 = ws.halo("stem", n, h2, w2, 64)
        _cg(ws, stem_mat, pc[f"{prefix}.conv1"], n, h2, w2, s1, relu=True, round_tf32=True)
        h, w = H // 4, W // 4
        x = ws.halo("pool", n, h, w, 64)
        ops.maxpool3x3s2(s1, n, h2, w2, x)
        cin = 64
        for li, (lname, planes, blocks, stride) in enumerate(zip(lnames, planes_t, blocks_t, strides_t)):
            for b in range(blocks):
                s = stride if b == 0 else 1
                d = 1 if dilation_t is None else dilation_t[li][0 if b == 0 else 1]
                ho, wo = h // s, w // s
                last = b == blocks - 1
                if last and li in keep:
                    out = keep[li]
                else:
                    out = ws.halo("blk%d" % (b & 1), n, ho, wo, 4 * planes)
                self._bottleneck(f"{prefix}.{lname}.{b}", x, n, h, w, cin, planes, s, b == 0, out, ws, dilation=d)
                x, h, w, cin = out, ho, wo, 4 * planes
        return x


class PropagationEngine(_ResNetTrunk):
    def __init__(self, state_dict: Dict[str, torch.Tensor], device, top_k: Optional[int],
                 act_dtype: Optional[torch.dtype] = None):
        self.device = torch.device(device)
        self.top_k = top_k
        self.act_dtype = act_dtype or act_dtype_from_env()
        # per-frame (sequential) work: memory read, decoder tail, memorize.  One workspace per LANE: lane 0 is
        # the default; a second lane exists when the forward and backward pass of one interaction run
        # concurrently on two streams (InferenceCore.interact), each with its own buffers and graphs.
        self.ws = Workspace(self.device, self.act_dtype)
        self._ws_lanes = {0: self.ws}
        # batched query pass — may run concurrently on another stream
        self.ws_q = Workspace(self.device, self.act_dtype)
        self.pc: Dict[str, PackedConv] = {}
        self._pack(state_dict)
        self.memread_algo = ops.MEMREAD_AUTO

    @contextlib.contextmanager
    def lane(self, i: int):
        """Context manager: the sequential-step workspace of lane i becomes `self.ws` (eager launches and graph
        CAPTURE bind buffer addresses; replay does not touch the engine)."""
        if i not in self._ws_lanes:
            self._ws_lanes[i] = Workspace(self.device, self.act_dtype)
        prev, self.ws = self.ws, self._ws_lanes[i]
        try:
            yield
        finally:
            self.ws = prev

    # ------------------------------------------------------------------ packing
    def _pack(self, sd):
        dev = self.device

        def conv(name, bn=None, stride=1, im2col=False, stem_s2d=False):
            self.pc[name] = ops.pack_conv(sd[name + ".weight"], sd.get(name + ".bias"),
                                          bn=_bn_of(sd, bn) if bn else None, stride=stride, im2col=im2col, device=dev,
                                          dtype=self.act_dtype, stem_s2d=stem_s2d)

        for prefix, lnames in (("mask_rgb_encoder", arch.MASK_LAYERS), ("rgb_encoder", arch.RGB_LAYERS)):
            # 7x7/2 stems: space-to-depth gather + four vertical taps (13 / 27 MB matrix instead of 54 MB of im2col)
            conv(f"{prefix}.conv1", bn=f"{prefix}.bn1", stride=2, stem_s2d=True)
            for lname, blocks, stride in zip(lnames, arch.TRUNK_BLOCKS, arch.TRUNK_STRIDES):
                for b in range(blocks):
                    p = f"{prefix}.{lname}.{b}"
                    s = stride if b == 0 else 1
                    conv(f"{p}.conv1", bn=f"{p}.bn1")
                    conv(f"{p}.conv2", bn=f"{p}.bn2", stride=s, im2col=(s == 2))
                    conv(f"{p}.conv3", bn=f"{p}.bn3")
                    if b == 0:
                        conv(f"{p}.downsample.0", bn=f"{p}.downsample.1", stride=s, im2col=True)
        for kv in ("kv_m_f16", "kv_q_f16"):
            # key and value projections read the same input: one GEMM with 640 output channels
            w = torch.cat([sd[f"{kv}.key_proj.weight"], sd[f"{kv}.val_proj.weight"]], 0)
            b = torch.cat([sd[f"{kv}.key_proj.bias"], sd[f"{kv}.val_proj.bias"]], 0)
            self.pc[kv] = ops.pack_conv(w, b, device=dev, dtype=self.act_dtype)
        self.has_decoder = "decoder.pred.weight" in sd  # AttentionReadNetwork: encoders + key/value heads only
        if self.has_decoder:
            for ent in arch.resblock_entries("decoder.compress", 1024, 512) + \
                    arch.upblock_entries("decoder.up_16_8", 512, 512, 256) + \
                    arch.upblock_entries("decoder.up_8_4", 256, 256, 256) + [("conv", "decoder.pred", 1, 256, 3, True)]:
                conv(ent[1])

    # ------------------------------------------------------------------ encoders
    def new_query_states(self, H: int, W: int, n: int = 1, keep_features: bool = False):
        """n QueryStates backed by ONE batched allocation each (kv, qk, s8, s4 [+ f16, f8, f4]); state i
        is the contiguous slice i, itself a valid batch-1 HALO map."""
        dev, dt = self.device, self.act_dtype
        h16, w16 = H // 16, W // 16
        kv = ops.halo_zeros(n, h16, w16, 640, dev)  # keys / values stay fp32 (they feed the bank and the read)
        qk = torch.empty((n, h16 * w16, 128), dtype=torch.float32, device=dev)
        s8 = ops.halo_zeros(n, H // 8, W // 8, 512, dev, dt)
        s4 = ops.halo_zeros(n, H // 4, W // 4, 256, dev, dt)
        f16 = ops.halo_zeros(n, h16, w16, 1024, dev, dt) if keep_features else None
        f8 = ops.halo_zeros(n, H // 8, W // 8, 512, dev, dt) if keep_features else None
        f4 = ops.halo_zeros(n, H // 4, W // 4, 256, dev, dt) if keep_features else None
        states = [QueryState(kv=kv[i:i + 1], qk=qk[i], s8=s8[i:i + 1], s4=s4[i:i + 1], h=H, w=W,
                             f16=None if f16 is None else f16[i:i + 1], f8=None if f8 is None else f8[i:i + 1],
                             f4=None if f4 is None else f4[i:i + 1]) for i in range(n)]
        batch = QueryState(kv=kv, qk=qk, s8=s8, s4=s4, h=H, w=W, f16=f16, f8=f8, f4=f4)
        return states, batch

    def new_query_state(self, H: int, W: int, keep_features: bool = False) -> QueryState:
        return self.new_query_states(H, W, 1, keep_features)[0][0]

    def _skip_path(self, p, skip, n, h, w, c, out):
        """skip_conv2(skip_conv1(skip_f)) of an UpsampleBlock (modules.py:101) for a batch of frames."""
        ws = self.ws_q
        s1 = ws.halo("sk_s1", n, h, w, c)
        s1r = ws.halo("sk_s1r", n, h, w, c)
        _cg(ws, skip, self.pc[f"{p}.skip_conv1"], n, h, w, s1, out_relu=s1r)
        return self._resblock(f"{p}.skip_conv2", s1, s1r, n, h, w, c, c, out, ws=ws)

    def encode_query_batch(self, frames: torch.Tensor, batch: QueryState) -> None:
        """get_query_values (prop_net.py:164-168) + the decoder skip paths for N frames at once
        (`frames` [N,3,H,W] on the device, `batch` the batched QueryState from new_query_states).
        Batching multiplies the tile count of the 1/8- and 1/16-resolution layers by N, which is
        what fills the 132 SMs."""
        N, _, H, W = frames.shape
        assert H % 16 == 0 and W % 16 == 0, "frames must be padded to multiples of 16 (pad_divide_by)"
        ws = self.ws_q
        pcs = self.pc["rgb_encoder.conv1"]
        stem = ws.mat("stem_q", N * (H // 2 + 2) * (W // 2 + 2), pcs.cin_pad)
        ops.stem_gather(frames, None, stem, s2d=True)
        h16, w16 = H // 16, W // 16
        f16 = batch.f16 if batch.f16 is not None else ws.halo("q_f16", N, h16, w16, 1024)
        f8 = batch.f8 if batch.f8 is not None else ws.halo("q_f8", N, H // 8, W // 8, 512)
        f4 = batch.f4 if batch.f4 is not None else ws.halo("q_f4", N, H // 4, W // 4, 256)
        self._trunk("rgb_encoder", arch.RGB_LAYERS, stem, N, H, W, {0: f4, 1: f8, 2: f16}, ws)
        _cg(ws, f16, self.pc["kv_q_f16"], N, h16, w16, batch.kv)
        ops.halo_to_pixels(batch.kv, N, h16, w16, 0, 128, batch.qk)  # pixel-major keys for the memory read
        if self.has_decoder:
            self._skip_path("decoder.up_16_8", f8, N, H // 8, W // 8, 512, batch.s8)
            self._skip_path("decoder.up_8_4", f4, N, H // 4, W // 4, 256, batch.s4)

    def encode_query(self, frame: torch.Tensor, qs: Optional[QueryState] = None, keep_features: bool = False) -> QueryState:
        """Single-frame query pass into `qs` (allocated when None)."""
        H, W = frame.shape[-2:]
        if qs is None:
            qs = self.new_query_state(H, W, keep_features)
        self.encode_query_batch(frame.reshape(1, 3, H, W), qs)
        return qs

    def encode_memory(self, frames: torch.Tensor, masks: torch.Tensor, objs: Optional[Tuple[int, int]] = None,
                      first: Optional[torch.Tensor] = None, maps: int = 0) -> torch.Tensor:
        """memorize (prop_net.py:144-162) of one clip (frame [1,3,H,W], masks [K,1,H,W]) or of C clips (frames
        [C,3,H,W], masks [C,K,1,H,W], any clip stride): returns the HALO [C*K,H/16,W/16,640] key|value map, clip-major
        (a workspace buffer: consume before the next call).  The "others" channel sums over the objects of the SAME
        clip: the stem gather takes the C (frame, K masks) groups in one launch.  `objs` (k0, n), one clip only:
        objects [k0, k0 + n) alone ([n,...] map), their "others" channels still summed over all K masks.
        `first` (object groups: C clips of different object counts): masks are the packed planes [maps + C,1,H,W]
        (each clip's background plane, then its objects), clip g owns maps [first[g], first[g+1])."""
        H, W = masks.shape[-2:]
        N = maps if first is not None else masks.shape[:-3].numel()  # K, or C*K
        pcs = self.pc["mask_rgb_encoder.conv1"]
        if first is not None:
            stem = self.ws.mat("stem_m", N * (H // 2 + 2) * (W // 2 + 2), pcs.cin_pad)
            ops.stem_gather_groups(frames, masks, N, first, stem)
        elif objs is None or objs == (0, N):
            stem = self.ws.mat("stem_m", N * (H // 2 + 2) * (W // 2 + 2), pcs.cin_pad)
            ops.stem_gather(frames.reshape(-1, 3, H, W), masks, stem, s2d=True)
        else:
            k0, N = objs
            stem = self.ws.mat("stem_m", N * (H // 2 + 2) * (W // 2 + 2), pcs.cin_pad)
            ops.stem_gather_range(frames, masks, k0, N, stem)
        f16 = self._trunk("mask_rgb_encoder", arch.MASK_LAYERS, stem, N, H, W, {}, self.ws)
        h16, w16 = H // 16, W // 16
        kv = self.ws.halo("kv_m", N, h16, w16, 640, torch.float32)
        _cg(self.ws, f16, self.pc["kv_m_f16"], N, h16, w16, kv)
        return kv

    def memorize_into(self, frames: torch.Tensor, masks: torch.Tensor, bank_k, bank_v, t: int, dyn_t=None,
                      dyn_sets: bool = False, first: Optional[torch.Tensor] = None) -> None:
        """encode_memory + bank_write into bank frame `t` (or the device scalar dyn_t, t its largest value) for every
        object: C clips of K <= CHUNK_OBJECTS objects in one batch, one clip of more objects in object_chunks.
        dyn_sets (C clips, masks [C,K,1,H,W]): dyn_t holds one frame per clip, clip c writes frame dyn_t[c].
        `first` (object groups): masks the packed planes [N + C,1,H,W] of C clips of different object counts, bank
        rows [0, N); clip g writes frame dyn_t[g]."""
        H, W = masks.shape[-2:]
        if first is not None:
            N = bank_k.shape[0]
            kv = self.encode_memory(frames, masks, first=first, maps=N)
            ops.bank_write_groups(kv, N, H // 16, W // 16, 0, 128, bank_k, bank_v, t, dyn_t, first)
            return
        N = masks.shape[:-3].numel()
        if dyn_sets:
            kv = self.encode_memory(frames, masks)
            ops.bank_write_sets(kv, N, masks.shape[0], H // 16, W // 16, 0, 128, bank_k, bank_v, t, dyn_t)
            return
        for k0, n in ([(0, N)] if masks.dim() == 5 else object_chunks(N)):
            kv = self.encode_memory(frames, masks, (k0, n))
            ops.bank_write(kv, n, H // 16, W // 16, 0, 128, bank_k[k0:k0 + n], bank_v[k0:k0 + n], t, dyn_t=dyn_t)

    # ------------------------------------------------------------------ decoder
    def _resblock(self, p, x_raw, x_relu, n, h, w, cin, cout, out, *, out_relu_only=False, out_relu=None, ws=None):
        """ResBlock (modules.py:28-35): out = (downsample(x) | x) + conv2(relu(conv1(relu(x))))."""
        ws = ws or self.ws
        pc = self.pc
        r = ws.halo("rb_r", n, h, w, cout)
        _cg(ws, x_relu, pc[f"{p}.conv1"], n, h, w, r, relu=True, round_tf32=True)
        res = x_raw
        if cin != cout:
            res = ws.halo("rb_ds", n, h, w, cout)
            _cg(ws, x_raw, pc[f"{p}.downsample"], n, h, w, res)
        _cg(ws, r, pc[f"{p}.conv2"], n, h, w, out, residual=res, relu=out_relu_only, out_relu=out_relu,
                      round_tf32=out_relu_only)
        return out

    @property
    def min_live_slots(self) -> int:
        """Fewest live bank slots a read accepts: top_k for the top-k read (as torch.topk), 1 for the dense read."""
        return 1 if self.top_k is None else self.top_k

    def _memory_read(self, bank_k, bank_v, slots: int, qk, n: int, cat, h16: int, w16: int, dyn_slots, q_div: int,
                     dyn_sets: bool = False, first: Optional[torch.Tensor] = None):
        """The memory read of n objects into channels [0, 512) of `cat`: the top-k read (prop_net.py:47-73) for
        top_k <= 64, the wide top-k read above that, or the dense read of the reference's top_k=None
        (prop_net.py:99-102).  The only place that tells them apart.  dyn_sets: qk [sets,hw,128] and one live slot
        count per set in dyn_slots (the per-set forms).  `first`: qk [groups,hw,128], one count per group, and the
        group table (the grouped forms)."""
        hw = h16 * w16
        if first is not None:
            nf = self.ws.full(n)
            if self.top_k is None:
                wsp = self.ws.raw("memread_dense", ops.memory_read_dense_workspace_bytes(nf, bank_k.shape[1], hw))
                ops.memory_read_dense_groups(bank_k, bank_v, slots, qk, cat, dyn_slots, first, halo_hw=(h16, w16),
                                             workspace=wsp)
            elif self.top_k > ops.TOPK_READ_MAX_K:
                wsp = self.ws.raw("memread_wide",
                                  ops.memory_read_wide_workspace_bytes(nf, bank_k.shape[1], hw, self.top_k))
                ops.memory_read_wide_groups(bank_k, bank_v, slots, qk, self.top_k, cat, dyn_slots, first,
                                            halo_hw=(h16, w16), workspace=wsp)
            else:
                wsp = self.ws.raw("memread", ops.memory_read_workspace_bytes(nf, slots, hw, self.top_k))
                ops.memory_read_groups(bank_k, bank_v, slots, qk, self.top_k, cat, dyn_slots, first, halo_hw=(h16, w16),
                                       workspace=wsp, algo=self.memread_algo)
            return
        if dyn_sets:
            nf = self.ws.full(n)  # a prefix batch reads through the full batch's workspace
            if self.top_k is None:
                wsp = self.ws.raw("memread_dense", ops.memory_read_dense_workspace_bytes(nf, bank_k.shape[1], hw))
                ops.memory_read_dense_sets(bank_k, bank_v, slots, qk, cat, dyn_slots, halo_hw=(h16, w16), workspace=wsp)
            elif self.top_k > ops.TOPK_READ_MAX_K:
                wsp = self.ws.raw("memread_wide",
                                  ops.memory_read_wide_workspace_bytes(nf, bank_k.shape[1], hw, self.top_k))
                ops.memory_read_wide_sets(bank_k, bank_v, slots, qk, self.top_k, cat, dyn_slots, halo_hw=(h16, w16),
                                          workspace=wsp)
            else:
                wsp = self.ws.raw("memread", ops.memory_read_workspace_bytes(nf, slots, hw, self.top_k))
                ops.memory_read_sets(bank_k, bank_v, slots, qk, self.top_k, cat, dyn_slots, halo_hw=(h16, w16),
                                     workspace=wsp, algo=self.memread_algo)
            return
        if self.top_k is None:
            wsp = self.ws.raw("memread_dense", ops.memory_read_dense_workspace_bytes(n, bank_k.shape[1], hw))
            ops.memory_read_dense(bank_k, bank_v, slots, qk, cat, out_coff=0, halo_hw=(h16, w16), workspace=wsp,
                                  dyn_slots=dyn_slots, q_div=q_div)
        elif self.top_k > ops.TOPK_READ_MAX_K:
            if self.top_k > ops.WIDE_READ_MAX_K:
                raise MivosError(f"memory read: top_k {self.top_k} exceeds the largest served top_k "
                                 f"({ops.WIDE_READ_MAX_K})")
            wsp = self.ws.raw("memread_wide", ops.memory_read_wide_workspace_bytes(n, bank_k.shape[1], hw, self.top_k))
            ops.memory_read_wide(bank_k, bank_v, slots, qk, self.top_k, cat, out_coff=0, halo_hw=(h16, w16),
                                 workspace=wsp, dyn_slots=dyn_slots, q_div=q_div)
        else:
            wsp = self.ws.raw("memread", ops.memory_read_workspace_bytes(n, slots, hw, self.top_k))
            ops.memory_read(bank_k, bank_v, slots, qk, self.top_k, cat, out_coff=0, halo_hw=(h16, w16), workspace=wsp,
                            algo=self.memread_algo, dyn_slots=dyn_slots, q_div=q_div)

    def segment(self, bank_k, bank_v, slots: int, q: QueryState, K: int, C: int = 1, *, prob_out=None, want_raw=False,
                want_prob=True, dyn_slots=None, dyn_sets: bool = False, first: Optional[torch.Tensor] = None):
        """segment_with_query (prop_net.py:170-181) + aggregate_wbg(keep_bg=True) (inference_core.py:175) for C
        clips.  The C*K object maps (clip-major: map c*K + k is object k of clip c) go through every convolution as
        ONE batch — the 1/16- and 1/8-resolution layers of a single clip have 14-54 row tiles for 132 SMs — while the
        operators whose operands differ per clip (memory read, skip broadcast, aggregation) take the C clips as groups
        of one launch.  One clip of more than CHUNK_OBJECTS objects runs the read and the decoder per object chunk
        (object_chunks), each chunk writing its slice of one K-object logits map; one aggregation over all K follows.
        bank_k/bank_v [C*K, cap, 128/512]; `q` the QueryState of one clip's frame, or for C > 1 the batched state of
        the C current frames (new_query_states(H, W, C)).  Returns (raw sigmoid [C*K,1,H,W] | None, prob
        [(K+1),1,H,W] | None), prob [C,K+1,1,H,W] for C > 1.  dyn_sets: `q` is a batched state of C >= 1 clips and
        dyn_slots holds one live slot count per clip (the per-set read).  `first` (object groups, C clips of
        different object counts): K is the number of object maps, clip g owns maps [first[g], first[g+1]) and the
        device table `first` [C+1] is read at run time; prob_out is the packed [K + C,1,H,W] (each clip's background
        plane, then its objects).  Returns (None, prob_out)."""
        H, W = q.h, q.w
        if first is not None:
            lg = self._decode(bank_k, bank_v, slots, q, K, C, dyn_slots, None, first=first)
            return ops.upsample4x_sigmoid_aggregate_groups(lg, K, H // 4, W // 4, first, prob_out=prob_out)
        chunks = object_chunks(K) if C == 1 else [(0, K)]
        if dyn_sets:
            lg = self._decode(bank_k, bank_v, slots, q, K, C, dyn_slots, None, dyn_sets=True)
        elif len(chunks) == 1:
            lg = self._decode(bank_k, bank_v, slots, q, K, C, dyn_slots, None)
        else:
            lg = self.ws.halo("logit", K, H // 4, W // 4, 32, torch.float32)
            for k0, n in chunks:
                self._decode(bank_k[k0:k0 + n], bank_v[k0:k0 + n], slots, q, n, 1, dyn_slots, lg[k0:k0 + n])
        return ops.upsample4x_sigmoid_aggregate_any(lg, K, H // 4, W // 4, want_raw=want_raw, want_prob=want_prob,
                                                    prob_out=prob_out, groups=C)

    def _decode(self, bank_k, bank_v, slots: int, q: QueryState, K: int, C: int, dyn_slots, lg, dyn_sets: bool = False,
                first: Optional[torch.Tensor] = None):
        """Memory read and decoder of C*K object maps as one batch; returns their decoder.pred logits in `lg` (a
        workspace map when None).  `first` (object groups): K is the number of maps, clip g owns [first[g], first[g+1])."""
        ws, pc = self.ws, self.pc
        H, W = q.h, q.w
        h16, w16 = H // 16, W // 16
        N = K if first is not None else C * K
        cat = ws.halo("cat", N, h16, w16, 1024)
        # ONE read for the C clips: object c*K + k reads query set c (q_div = K objects per set; one clip: q_div 0)
        self._memory_read(bank_k, bank_v, slots, q.qk, N, cat, h16, w16, dyn_slots, K if C > 1 else 0, dyn_sets, first)
        if first is not None:
            ops.halo_copy_groups(q.kv, cat, N, h16, w16, 512, first, src_coff=128, dst_coff=512)
        else:
            ops.halo_copy(q.kv, cat, N, h16, w16, 512, src_coff=128, dst_coff=512)  # cat([readout, v16]) :178-179
        catr = ws.halo("catr", N, h16, w16, 1024)
        ops.halo_copy(cat, catr, N, h16, w16, 1024, relu=True)
        x16 = ws.halo("dec16", N, h16, w16, 512)
        self._resblock("decoder.compress", cat, catr, N, h16, w16, 1024, 512, x16)
        # up_16_8 / up_8_4 (modules.py:100-104): the skip paths were produced by the query pass (q.s8 / q.s4, one map
        # per clip); the reference broadcasts them over the objects in the add
        x8 = ws.halo("dec8", N, H // 8, W // 8, 256)
        self._upblock_tail("decoder.up_16_8", q.s8, x16, N, H // 8, W // 8, 512, 256, x8, final_relu=False, first=first)
        x4 = ws.halo("dec4", N, H // 4, W // 4, 256)
        self._upblock_tail("decoder.up_8_4", q.s4, x8, N, H // 4, W // 4, 256, 256, x4, final_relu=True, first=first)
        if lg is None:
            lg = ws.halo("logit", N, H // 4, W // 4, 32, torch.float32)
        _cg(ws, x4, pc["decoder.pred"], N, H // 4, W // 4, lg)
        return lg

    def _upblock_tail(self, p, s2_skip, up, K, h, w, up_c, out_c, out, final_relu, first=None):
        """x = skip (one map per frame, broadcast over that frame's objects) + bilinear_x2(up); out_conv ResBlock.
        `first`: the skip map of frame g is broadcast over the maps of object group g."""
        ws = self.ws
        s2 = ws.halo("ub_s2", K, h, w, up_c)
        s2r = ws.halo("ub_s2r", K, h, w, up_c)
        if first is not None:
            ops.upsample2x_add_groups(s2, up, K, h, w, s2_skip, first, x_relu=s2r)
        else:
            ops.upsample2x_add(s2, up, K, h, w, x_relu=s2r, skip=s2_skip)
        return self._resblock(f"{p}.out_conv", s2, s2r, K, h, w, up_c, out_c, out, out_relu_only=final_relu)


class FusionEngine:
    """FusionNet.forward (model/fusion_net.py:32-50) on a HALO (1,H,W,32) map."""

    def __init__(self, state_dict, device):
        self.device = torch.device(device)
        self.ws = Workspace(self.device)
        self.pc = {e[1]: ops.pack_conv(state_dict[e[1] + ".weight"], state_dict[e[1] + ".bias"], device=self.device)
                   for e in arch.fusion_entries()}

    def forward_logit_halo(self, im, seg1, seg2, attn, nc: float, nr: float) -> Tuple[torch.Tensor, int, int]:
        H, W = im.shape[-2:]
        ws, pc = self.ws, self.pc
        x0 = ws.halo("in", 1, H, W, 32)
        ops.fusion_gather(im, seg1, seg2, attn, nc, nr, x0)
        x = ws.halo("x", 1, H, W, 32)
        _cg(ws, x0, pc["conv1.0"], 1, H, W, x, relu=True, round_tf32=True)
        r = ws.halo("r", 1, H, W, 32)
        _cg(ws, x, pc["conv2.0"], 1, H, W, r, relu=True, round_tf32=True)
        y = ws.halo("y", 1, H, W, 32)
        _cg(ws, r, pc["conv2.2"], 1, H, W, y, residual=x, relu=True, round_tf32=True)
        _cg(ws, y, pc["conv3.0"], 1, H, W, r, relu=True, round_tf32=True)
        _cg(ws, r, pc["conv3.2"], 1, H, W, x, residual=y, relu=True, round_tf32=True)
        lg = ws.halo("lg", 1, H, W, 32)
        _cg(ws, x, pc["final_conv"], 1, H, W, lg)
        return lg, H, W


class S2MEngine(_ResNetTrunk):
    """Scribble-to-Mask network (SURVEY.md 8f-3): DeepLabV3+ on a 6-channel ResNet-50 at output stride
    16 (model/s2m/s2m_network.py:8-33, s2m_resnet.py:70-148, _deeplab.py:30-58,119-160), for a batch of
    n inputs (one per object of an interaction: davis_processor.py:55-68, s2m_controller.py:28-35).

    Every convolution is a wgmma implicit GEMM (mivos_conv_gemm); BatchNorm is folded at pack time;
    the dilated 3x3 convs (layer4 blocks 1-2, the three ASPP branches) read a dilated gather; the
    image-pooling branch is pooled and broadcast BEFORE its 1x1 conv (the conv, BN and ReLU commute
    with broadcasting a constant map), so that its output lands straight in the 1280-channel concat
    buffer like the other four branches; torch.cat never happens — producers write channel windows."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device, act_dtype: Optional[torch.dtype] = None):
        self.device = torch.device(device)
        self.act_dtype = act_dtype or act_dtype_from_env()
        self.ws = Workspace(self.device, self.act_dtype)
        self.pc: Dict[str, PackedConv] = {}
        sd, dev, dt = state_dict, self.device, self.act_dtype

        def conv(name, bn, stride=1, im2col=False):
            self.pc[name] = ops.pack_conv(sd[name + ".weight"], sd.get(name + ".bias"),
                                          bn=_bn_of(sd, bn) if bn else None, stride=stride, im2col=im2col, device=dev, dtype=dt)

        conv("backbone.conv1", "backbone.bn1", stride=2, im2col=True)
        for lname, blocks, stride, dil in zip(arch.S2M_LAYERS, arch.S2M_BLOCKS, arch.S2M_STRIDES, arch.S2M_DILATION):
            for b in range(blocks):
                p = f"backbone.{lname}.{b}"
                s = stride if b == 0 else 1
                d = dil[0 if b == 0 else 1]
                conv(f"{p}.conv1", f"{p}.bn1")
                conv(f"{p}.conv2", f"{p}.bn2", stride=s, im2col=(s == 2 or d > 1))
                conv(f"{p}.conv3", f"{p}.bn3")
                if b == 0:
                    conv(f"{p}.downsample.0", f"{p}.downsample.1", stride=s, im2col=True)
        c = "classifier"
        conv(f"{c}.project.0", f"{c}.project.1")
        conv(f"{c}.aspp.convs.0.0", f"{c}.aspp.convs.0.1")
        for i in range(1, 4):
            conv(f"{c}.aspp.convs.{i}.0", f"{c}.aspp.convs.{i}.1", im2col=True)
        conv(f"{c}.aspp.convs.4.1", f"{c}.aspp.convs.4.2")
        conv(f"{c}.aspp.project.0", f"{c}.aspp.project.1")
        conv(f"{c}.classifier.0", f"{c}.classifier.1")
        conv(f"{c}.classifier.3", None)

    def logits_halo(self, x: torch.Tensor):
        """x [n,6,H,W] fp32 on the device (H, W multiples of 16) -> (fp32 HALO logits (n,H/4,W/4,32),
        channel 0 = classifier output at 1/4 resolution — _deeplab.py:52 —, n, H, W)."""
        n, cin, H, W = x.shape
        assert cin == 6 and H % 16 == 0 and W % 16 == 0, "S2M input: [n,6,H,W], H and W multiples of 16 (pad_divide_by)"
        ws, pc = self.ws, self.pc
        stem = ws.mat("stem", n * (H // 2 + 2) * (W // 2 + 2), pc["backbone.conv1"].cin_pad)
        if ops.stem_frames_untiled(cin, W, stem.dtype == torch.float16):
            ops.stem_gather_frames(x, stem)
        else:  # wider than 7 staged input rows fit in shared memory: 1378 px in fp32, 2762 in fp16
            ops.stem_gather_frames_tiled(x, stem)
        h4, w4, h16, w16 = H // 4, W // 4, H // 16, W // 16
        low = ws.halo("low", n, h4, w4, 256)
        f = self._trunk("backbone", arch.S2M_LAYERS, stem, n, H, W, {0: low}, ws, planes_t=arch.S2M_PLANES,
                        blocks_t=arch.S2M_BLOCKS, strides_t=arch.S2M_STRIDES, dilation_t=arch.S2M_DILATION)
        # ---- ASPP (_deeplab.py:141-160): five branches write 256-channel windows of one map
        c = "classifier"
        cat = ws.halo("aspp_cat", n, h16, w16, 1280)
        _cg(ws, f, pc[f"{c}.aspp.convs.0.0"], n, h16, w16, cat, out_coff=0, relu=True, round_tf32=True)
        g = ws.mat("aspp_g", n * (h16 + 2) * (w16 + 2), 9 * 2048)
        for i, rate in enumerate(arch.S2M_ASPP_RATES, start=1):
            ops.gather_dilated(f, n, h16, w16, 2048, rate, g)
            _cg(ws, g, pc[f"{c}.aspp.convs.{i}.0"], n, h16, w16, cat, out_coff=256 * i, relu=True, round_tf32=True)
        pooled = ws.halo("aspp_pool", n, h16, w16, 2048)
        ops.halo_avgpool_broadcast(f, n, h16, w16, 2048, pooled)
        _cg(ws, pooled, pc[f"{c}.aspp.convs.4.1"], n, h16, w16, cat, out_coff=1024, relu=True, round_tf32=True)
        proj = ws.halo("aspp_proj", n, h16, w16, 256)
        _cg(ws, cat, pc[f"{c}.aspp.project.0"], n, h16, w16, proj, relu=True, round_tf32=True)
        # ---- V3+ head (_deeplab.py:48-52): [low-level 48 | ASPP x4 256 | zero pad to 320]
        head = ws.halo("head_cat", n, h4, w4, 320)
        _cg(ws, low, pc[f"{c}.project.0"], n, h4, w4, head, out_coff=0, relu=True, round_tf32=True)
        ops.upsample_bilinear(proj, n, h16, w16, head, h4, w4, 256, dst_coff=48)
        y = ws.halo("head_y", n, h4, w4, 256)
        _cg(ws, head, pc[f"{c}.classifier.0"], n, h4, w4, y, relu=True, round_tf32=True)
        lg = ws.halo("logit", n, h4, w4, 32, torch.float32)
        _cg(ws, y, pc[f"{c}.classifier.3"], n, h4, w4, lg)
        return lg, n, H, W

    def forward(self, x: torch.Tensor, sigmoid: bool = False, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[n,6,H,W] -> logits (or probabilities) [n,1,H,W]: utils.py:16-21 (+ the callers' torch.sigmoid)."""
        lg, n, H, W = self.logits_halo(x)
        return ops.halo_upsample_to_plane(lg, n, H // 4, W // 4, H, W, sigmoid=sigmoid, out=out)
