"""Drop-in ``PropagationNetwork`` (reference: model/propagation/prop_net.py:131-200).

Same constructor, same ``state_dict`` keys (597 tensors), same public methods and tensor
layouts at the boundary; every method runs hand-written sm_90a kernels through the C ABI.
Internally features stay in the HALO layout; the reference-layout (NCHW) entry points convert at
the boundary, while ``InferenceCore`` uses the ``*_resident`` methods that never leave HBM-native
layouts.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn as nn

from . import arch, ops
from . import _lib
from .engine import PropagationEngine, QueryState, act_dtype_from_env


class _Reader(nn.Module):
    """Parameter-less stand-in for EvalMemoryReader / AttentionMemory (prop_net.py:75-129): keeps
    the attribute surface (``net.memory.top_k``) of the reference."""

    def __init__(self, top_k):
        super().__init__()
        self.top_k = top_k
        self.km = None


class PropagationNetwork(nn.Module):
    def __init__(self, top_k: int = 50, act_dtype: Optional[torch.dtype] = None):
        """`act_dtype` (extension over the reference signature, prop_net.py:132): torch.float32 (TF32
        tensor-core path) or torch.float16; None reads MIVOS_ACT_DTYPE (engine.act_dtype_from_env)."""
        super().__init__()
        self.act_dtype = act_dtype
        g = torch.Generator().manual_seed(0)
        arch.build_param_tree(self, arch.propagation_entries(), g)
        self.memory = _Reader(top_k)
        self.attn_memory = _Reader(top_k)
        self._engine: Optional[PropagationEngine] = None
        self._engine_key = None
        self._engines = {}  # (device, top_k, act dtype) -> PropagationEngine
        self.eval()

    # ------------------------------------------------------------------ engine lifecycle
    def _tensor_signature(self):
        return tuple((t.data_ptr(), t.dtype, t.device) for t in list(self.parameters()) + list(self.buffers()))

    def _apply(self, fn, *a, **k):
        # parameters moved / cast: repack lazily.  A no-op .to(device) — every InferenceCore
        # construction does one (reference inference_core.py:24) — must NOT throw away the packed
        # weights, workspaces and captured graphs.
        before = self._tensor_signature()
        r = super()._apply(fn, *a, **k)
        if self._tensor_signature() != before:
            self._engine, self._engines = None, {}
        return r

    def load_state_dict(self, *a, **k):
        self._engine, self._engines = None, {}
        return super().load_state_dict(*a, **k)

    @property
    def top_k(self) -> int:
        return self.memory.top_k

    def engine(self) -> PropagationEngine:
        """The packed network for (device, top_k, activation type).  The activation type is the
        constructor's `act_dtype`, else MIVOS_ACT_DTYPE, else the CALLER'S precision context (fp16 under
        torch.autocast, TF32 otherwise — engine.act_dtype_from_env): one engine per type is kept, so a
        network driven both ways (GUI under autocast, evaluation in fp32) never repacks."""
        p = next(self.parameters())
        _lib.require_cuda_device(p.device, "PropagationNetwork")
        act = self.act_dtype or act_dtype_from_env()
        key = (p.device, self.memory.top_k, act)
        if self._engine is None or self._engine_key != key:
            eng = self._engines.get(key)
            if eng is None:
                sd = {k: v.detach().float() for k, v in self.state_dict().items()}
                eng = PropagationEngine(sd, p.device, self.memory.top_k, act_dtype=act)
                self._engines[key] = eng
            self._engine, self._engine_key = eng, key
        return self._engine

    @staticmethod
    def _f32(t: torch.Tensor) -> torch.Tensor:
        # callers may run under autocast / hand fp16 tensors (interactive_gui.py:990); tensors at the
        # reference-layout boundary are fp32, the engine converts to its own activation type
        return t.detach().float().contiguous()

    # ------------------------------------------------------------------ resident (HALO) API
    def encode_query_resident(self, frame: torch.Tensor, qs: Optional[QueryState] = None) -> QueryState:
        return self.engine().encode_query(self._f32(frame), qs)

    def encode_query_batch_resident(self, frames: torch.Tensor, batch: QueryState) -> None:
        """Query pass (trunk + key/value projection + decoder skip paths) for [N,3,H,W] frames into the
        batched QueryState from ``engine().new_query_states``."""
        self.engine().encode_query_batch(self._f32(frames), batch)

    def memorize_resident(self, frame: torch.Tensor, masks: torch.Tensor, bank_k: torch.Tensor, bank_v: torch.Tensor,
                          slot: int, dyn_slot: Optional[torch.Tensor] = None) -> None:
        """memorize() straight into BANK slot `slot` (slot-major keys/values).  `dyn_slot`: int32
        device scalar that overrides `slot` at run time (CUDA-graph replay)."""
        eng = self.engine()
        masks = self._f32(masks)
        K, _, H, W = masks.shape
        kv = eng.encode_memory(self._f32(frame), masks)
        ops.bank_write(kv, K, H // 16, W // 16, 0, 128, bank_k, bank_v, slot, dyn_t=dyn_slot)

    def segment_resident(self, bank_k, bank_v, slots: int, qs: QueryState, K: int, want_raw=False, want_prob=True,
                         prob_out=None, dyn_slots=None):
        return self.engine().segment(bank_k, bank_v, slots, qs, K, want_raw=want_raw, want_prob=want_prob,
                                     prob_out=prob_out, dyn_slots=dyn_slots)

    # ------------------------------------------------------------------ reference-layout API
    def memorize(self, frame: torch.Tensor, masks: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """prop_net.py:144-162 -> (k16 [K,128,1,h,w], v16 [K,512,1,h,w])."""
        eng = self.engine()
        masks = self._f32(masks)
        K, _, H, W = masks.shape
        kv = eng.encode_memory(self._f32(frame), masks)
        h, w = H // 16, W // 16
        k16 = ops.halo_to_nchw(kv, K, h, w, 128, coff=0)
        v16 = ops.halo_to_nchw(kv, K, h, w, 512, coff=128)
        return k16.unsqueeze(2), v16.unsqueeze(2)

    def get_query_values(self, frame: torch.Tensor):
        """prop_net.py:164-168 -> (f16, f8, f4, k16, v16) in NCHW."""
        qs = self.engine().encode_query(self._f32(frame), None, keep_features=True)
        H, W = qs.h, qs.w
        f16 = ops.halo_to_nchw(qs.f16, 1, H // 16, W // 16, 1024)
        f8 = ops.halo_to_nchw(qs.f8, 1, H // 8, W // 8, 512)
        f4 = ops.halo_to_nchw(qs.f4, 1, H // 4, W // 4, 256)
        k16 = ops.halo_to_nchw(qs.kv, 1, H // 16, W // 16, 128, coff=0)
        v16 = ops.halo_to_nchw(qs.kv, 1, H // 16, W // 16, 512, coff=128)
        return f16, f8, f4, k16, v16

    def segment_with_query(self, keys, values, f16, f8, f4, k16, v16) -> torch.Tensor:
        """prop_net.py:170-181 -> sigmoid probabilities [K,1,H,W] (no aggregation)."""
        eng = self.engine()
        keys, values = self._f32(keys), self._f32(values)
        K, _, T, h, w = keys.shape
        H, W = h * 16, w * 16
        dev = keys.device
        slots = T * h * w
        bank_k = torch.empty((K, slots, 128), dtype=torch.float32, device=dev)
        bank_v = torch.empty((K, slots, 512), dtype=torch.float32, device=dev)
        ops.bank_from_nchw(keys, values, bank_k, bank_v)
        qs = eng.new_query_state(H, W, keep_features=True)
        ops.nchw_to_halo(self._f32(f8), qs.f8)
        ops.nchw_to_halo(self._f32(f4), qs.f4)
        ops.nchw_to_halo(self._f32(k16), qs.kv, coff=0)
        ops.nchw_to_halo(self._f32(v16), qs.kv, coff=128)
        ops.halo_to_pixels(qs.kv, 1, h, w, 0, 128, qs.qk)
        # the skip paths run in the query-pass workspace (engine.ws_q): order them after any batched query pass a
        # session may have in flight on the network's side stream, and the side stream after them
        cur, side = torch.cuda.current_stream(dev), eng.__dict__.get("_qstream")
        if side is not None:
            cur.wait_stream(side)
        eng._skip_path("decoder.up_16_8", qs.f8, 1, H // 8, W // 8, 512, qs.s8)
        eng._skip_path("decoder.up_8_4", qs.f4, 1, H // 4, W // 4, 256, qs.s4)
        if side is not None:
            side.wait_stream(cur)
        raw, _ = eng.segment(bank_k, bank_v, slots, qs, K, want_raw=True, want_prob=False)
        return raw

    def get_W(self, mk16, qk) -> torch.Tensor:
        """prop_net.py:183 / AttentionMemory.forward (:115-129): mk16 [B,128,1,h,w], qk [1,128,h,w] ->
        W [B,hw,hw], softmax over the memory axis (dim 1), T = 1, no top-k."""
        mk16, qk = self._f32(mk16), self._f32(qk)
        b = mk16.shape[0]
        h, w = qk.shape[-2:]
        hw = h * w
        qpm = qk.reshape(128, hw).t().contiguous()
        return torch.stack([ops.attention_weights(mk16[i].reshape(128, hw).t().contiguous(), qpm) for i in range(b)], 0)

    def get_attention(self, mk16, pos_mask, neg_mask, qk16) -> torch.Tensor:
        """prop_net.py:187-200 -> [b,2,H,W] (b = 1 object per call, as in inference_core.py:212)."""
        mk16, qk16 = self._f32(mk16), self._f32(qk16)
        b = mk16.shape[0]
        h, w = qk16.shape[-2:]
        hw = h * w
        outs = []
        qpm = qk16.reshape(128, hw).t().contiguous()
        for i in range(b):
            mpm = mk16[i].reshape(128, hw).t().contiguous()
            outs.append(ops.attention_map(mpm, qpm, h, w, self._f32(pos_mask[i:i + 1]), self._f32(neg_mask[i:i + 1])))
        return outs[0] if b == 1 else torch.cat(outs, 0)

    def get_attention_resident(self, mk_pix: torch.Tensor, qs: QueryState, pos_mask, neg_mask) -> torch.Tensor:
        """Same as get_attention with the memory key already pixel-major [hw,128]."""
        return ops.attention_map(mk_pix, qs.qk, qs.h // 16, qs.w // 16, self._f32(pos_mask), self._f32(neg_mask))

    def forward(self, *a, **k):  # the reference module has no forward either
        raise NotImplementedError("use memorize / get_query_values / segment_with_query / get_attention")
