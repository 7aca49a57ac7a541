"""CPU: the oracle against outputs of the UNMODIFIED reference on inputs and seeds that are NOT the other
fixtures — the oracle is pinned to the reference itself on fresh data, not only to the vectors the other tests
use.  The reference's outputs were stored by oracle/gen_golden_live.py (tests/golden/reference_live*.npz).  Integer
outputs (masks, overlays, palette) must be identical; floating-point outputs agree to fp32 rounding, the tolerance of
the other golden tests (tests/test_oracle_golden.py): with the same torch build they are bit-identical on the CPU
that stored them, while another CPU's kernels may round the same convolutions differently in the last bits."""
import numpy as np
import pytest
import torch

TOL = 1e-5


def _close(a, b, tol=TOL):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return a.shape == b.shape and float((a - b).abs().max()) <= tol * max(1.0, float(b.abs().max()))


@pytest.fixture(scope="module")
def ref(golden):
    g = golden("reference_live.npz")
    return {k: torch.from_numpy(v) if v.dtype.kind == "f" else v for k, v in g.items()}


def test_propagation_ops_live(ref, prop_sd, fuse_sd):
    from oracle import stm_oracle as O, weights as Wt
    images, mask = Wt.synthetic_clip(3, 64, 96, 3, seed=2024)  # three objects: the "others" channel sums two masks
    frame = images[:, 1]
    for i, a in enumerate(O.get_query_values(prop_sd, frame)):
        assert _close(a, ref[f"ops_qv{i}"])
    mk, mv = ref["ops_mk"], ref["ops_mv"]
    ok, ov = O.memorize(prop_sd, frame, mask[1:])
    assert _close(ok, mk) and _close(ov, mv)
    qv = O.get_query_values(prop_sd, images[:, 2])
    for i, a in enumerate(qv):
        assert _close(a, ref[f"ops_qv2_{i}"])
    seg = ref["ops_seg"]
    assert _close(O.segment_with_query(prop_sd, mk, mv, *qv, top_k=20), seg)
    agg = ref["ops_agg"]
    assert _close(O.aggregate_wbg(seg, keep_bg=True), agg)
    assert float(np.abs(O.aggregate_wbg_f64(seg.numpy(), keep_bg=True) - agg.numpy()).max()) <= 5e-7
    pos, neg = (mask[1:2] - seg[0:1]).clamp(0, 1), (seg[0:1] - mask[1:2]).clamp(0, 1)
    at = ref["ops_att"]
    assert _close(O.get_attention(None, mk[0:1], pos, neg, qv[3]), at)
    assert float(np.abs(O.get_attention_f64(mk[0:1].numpy(), pos.numpy(), neg.numpy(), qv[3].numpy()) - at.numpy()).max()) <= 2e-6
    dist = torch.tensor([[0.25, 0.75]])
    assert _close(O.fusion_net(fuse_sd, images[:, 2], seg[0:1], agg[1:2], at, dist), ref["ops_fuse"])


def test_inference_core_live(ref, prop_sd, fuse_sd):
    """Whole interact() runs, two interactions (the second one fuses): bank trace is not observable in the
    reference, so probabilities (to fp32 rounding) and masks (on every decided pixel) are compared."""
    from oracle import stm_oracle as O, weights as Wt
    images, mask = Wt.synthetic_clip(7, 64, 88, 2, seed=77)  # 88 -> padded to 96
    oc = O.OracleInferenceCore(prop_sd, fuse_sd, images, 2, mem_freq=2, top_k=20)
    for j, (m, idx) in enumerate(((mask, 1), (mask.flip(-1).contiguous(), 6))):
        rm = ref[f"ic_masks{j}"]
        om = oc.interact(m, idx)
        rp = ref[f"ic_prob{j}"]
        assert rm.shape == om.shape == (7, 64, 88) and _close(rp, oc.prob)
        # every DECIDED pixel has the same label: where the reference's best object leads the runner-up by more than
        # twice the tolerance (an argmax can only flip inside that margin)
        left = (rp.shape[-1] - 88) // 2
        top2 = rp[:, :, 0, :, left:left + 88].topk(2, dim=0).values
        decided = ((top2[0] - top2[1]) > 2 * TOL).numpy()
        assert decided.mean() > 0.9 and (rm == om)[decided].all()
    assert _close(ref["ic_certain_mem_k"], oc.certain_mem_k)


def test_s2m_live(ref):
    from oracle import s2m_oracle as S, weights as Wt
    sd = Wt.make_s2m_state_dict()
    x = torch.randn((2, 6, 64, 80), generator=torch.Generator().manual_seed(5))
    assert _close(S.s2m_forward(sd, x), ref["s2m_logits"])
    image = torch.randn((1, 3, 64, 80), generator=torch.Generator().manual_seed(6))
    prev = torch.zeros((1, 64, 80), dtype=torch.int64)
    prev[:, 10:30, 10:40] = 1
    scr = np.full((60, 75), 255, dtype=np.uint8)  # unpadded: the controller pads the scribble maps
    scr[20:22, 5:50] = 1
    scr[40:42, 30:70] = 0
    assert _close(S.s2m_controller_interact(sd, image, prev, scr, 1), ref["s2m_ctrl"])


def test_egress_live(ref):
    from oracle import egress_oracle as EO
    assert np.array_equal(ref["egress_palette"], EO.color_map())
    rng = np.random.default_rng(9)
    image = rng.integers(0, 256, size=(40, 52, 3), dtype=np.uint8)
    mask = rng.integers(0, 7, size=(40, 52), dtype=np.uint8) * (rng.random((40, 52)) > 0.6)
    mask = mask.astype(np.uint8)
    for j, alpha in enumerate((0.5, 0.37)):
        assert np.array_equal(ref[f"egress_overlay{j}"], EO.overlay_davis(image, mask, alpha))
        assert np.array_equal(ref[f"egress_fade{j}"], EO.overlay_davis(image, mask, alpha, fade=True))


def test_fusion_generator_flow_live(ref, prop_sd):
    """SURVEY §8f-1: the client flow restated in tests/test_gpu_clients.py (what the GPU test drives our
    PropagationNetwork through) equals the reference's real FusionGenerator class."""
    import types
    from oracle import stm_oracle as O, weights as Wt
    from test_gpu_clients import fusion_generator_flow
    images, mask = Wt.synthetic_clip(5, 128, 168, 2, seed=31)
    soft = mask[1:] * 0.8 + 0.05
    api = types.SimpleNamespace(pad_divide_by=O.pad_divide_by, aggregate_wbg=O.aggregate_wbg,
                                memorize=lambda f, m: O.memorize(prop_sd, f, m),
                                get_query_values=lambda f: O.get_query_values(prop_sd, f),
                                segment_with_query=lambda *a: O.segment_with_query(prop_sd, *a, top_k=50))
    prob = fusion_generator_flow(api, images, soft, 2, 0, 4, mem_freq=2)  # [K+1, T, 1, nh, nw], padded 168 -> 176
    assert _close(prob[:, :, 0, :, 4:-4], ref["fg_prob"])  # reference: [K+1, T, h, w], unpadded


def test_attention_read_network_live(ref, prop_sd):
    """SURVEY §8f-2: AttentionReadNetwork.forward (model/attn_network.py:48-80) on a fresh batch."""
    from oracle import stm_oracle as O
    g = torch.Generator().manual_seed(123)
    image, query = torch.randn((1, 3, 48, 80), generator=g), torch.randn((1, 3, 48, 80), generator=g)
    m11, m21, m12, m22 = (torch.rand((1, 1, 48, 80), generator=g) for _ in range(4))
    o1, o2 = O.attention_read_network(prop_sd, image, m11, m21, m12, m22, query)
    assert _close(o1, ref["attn_a1"]) and _close(o2, ref["attn_a2"])
