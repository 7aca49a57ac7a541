"""GPU: the propagation-path elementwise, layout, attention and stem-gather kernels (csrc/elementwise.cu,
csrc/halo_ops.cu, csrc/attention.cu) at ragged shapes and edge inputs, against plain float64 statements of the same
operations; and the graph-staging kernels (store_i32, store_words, copy_segments) bit for bit.

Every reference is computed from the operands the kernel saw (fp16-rounded where the map is fp16; the kernel's
own fp32 intermediate output where a stage is checked on its own).  Copies, gathers, pooling and argmax are
bit-exact.  Arithmetic kernels get an elementwise bound derived from the kernel's fp32 operations; each bound is
written as a formula with its derivation, and every check prints its largest ratio of observed error to bound
(run with -s).  Outputs are pre-filled with a sentinel, and the sentinel must survive wherever a kernel writes
nothing: the HALO border, channels outside the window, pad columns of im2col rows, bank rows outside the written
slots.  Inputs a kernel must not read (HALO borders of bilinear sources, channels outside the window) hold NaN or
a sentinel, so a stray read shows up in the output."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from mivos_b200 import _lib, ops  # noqa: E402
from op_references import (CLAMP_HI, CLAMP_LO, GAMMA, H16, U, _bilinear, _sum_and_range,  # noqa: E402,F401
                           aggregate_reference, attention_reference, stem_images, stem_matrix)
from op_references import round16 as _round16  # noqa: E402

VEC = {torch.float32: 4, torch.float16: 8}  # elements per 16-byte vector
SENT = 7.0
NAN = float("nan")


def _check(what, got, ref, bound):
    """Elementwise |got - ref| <= bound; prints the largest ratio (NaN in `got` fails)."""
    err = (got.double() - ref).abs()
    ratio = float((err / bound).max())
    print(f"{what}: max err/bound = {ratio:.3g}")
    assert ratio <= 1.0, f"{what}: max err/bound = {ratio:.3g} (max err {float(err.max()):.3e})"


def _halo(x, cstride, coff=0, fill=0.0, border=None, dtype=torch.float32):
    """[n, c, h, w] -> HALO [n, h+2, w+2, cstride] holding x in channels [coff, coff + c); `fill` elsewhere,
    `border` (default `fill`) on the one-pixel border of every channel."""
    n, c, h, w = x.shape
    hb = torch.full((n, h + 2, w + 2, cstride), fill if border is None else border, dtype=dtype, device=x.device)
    hb[:, 1:-1, 1:-1, :] = fill
    hb[:, 1:-1, 1:-1, coff:coff + c] = x.permute(0, 2, 3, 1).to(dtype)
    return hb


# ------------------------------------------------------------------------------------------------ attention

def _attention_inputs(h16, w16, scale, seed, dev):
    g = torch.Generator().manual_seed(seed)
    hw = h16 * w16
    mk = (torch.randn(hw, 128, generator=g) * scale).to(dev)
    qk = (torch.randn(hw, 128, generator=g) * scale).to(dev)
    pos = torch.rand(1, 1, 16 * h16, 16 * w16, generator=g).to(dev)
    neg = torch.rand(1, 1, 16 * h16, 16 * w16, generator=g).to(dev)
    return mk, qk, pos, neg


def test_attention_smem_limit_never_lowered(dev):
    """attention_map and attention_weights launch one kernel with 4096 + 32 hw bytes of dynamic shared memory.
    attention_weights at hw = 6904 (8 x 863) asks for 256 B less than attention_map at hw = 6912 (64 x 108), and
    for more than any attention_weights call that runs before this test (the rest of the suite calls get_W at
    hw = 48 only; this test comes first in its file).  Had the two entry points each kept their own record of the
    kernel's limit, the middle call would lower it and the third call would be refused at launch."""
    mk, qk, pos, neg = _attention_inputs(64, 108, 1.0, 11, dev)
    mk2, qk2 = mk[:6904].contiguous(), qk[:6904].contiguous()
    first = ops.attention_map(mk, qk, 64, 108, pos, neg)
    W2 = ops.attention_weights(mk2, qk2)
    third = ops.attention_map(mk, qk, 64, 108, pos, neg)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    _, _, out, outb = attention_reference(mk, qk, 64, 108, pos, neg)
    _check("attention_map hw=6912 before get_W", first, out, outb)
    _check("attention_map hw=6912 after get_W hw=6904", third, out, outb)
    del out, outb
    Wr, Wb = attention_reference(mk2, qk2)
    _check("attention_weights hw=6904", W2, Wr, Wb)


@pytest.mark.parametrize("scale", [1.0, 4.0])  # x4: logits of std 16, peaked columns where the max subtraction matters
@pytest.mark.parametrize("h16,w16", [(1, 1), (7, 9), (5, 13), (17, 83), (64, 108)])
def test_attention_ragged(dev, h16, w16, scale):
    """hw = 1 (no bilinear neighbour), 63 and 65 (ragged last CTA of 8 queries), 1411 (above the default 48 KB of
    shared memory, so it needs the opt-in attribute; ragged last CTA), 6912 (the 220 KB limit)."""
    hw = h16 * w16
    mk, qk, pos, neg = _attention_inputs(h16, w16, scale, hw * 10 + int(scale), dev)
    out = ops.attention_map(mk, qk, h16, w16, pos, neg)
    W = ops.attention_weights(mk, qk)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    Wr, Wb, outr, outb = attention_reference(mk, qk, h16, w16, pos, neg)
    _check(f"attention_weights hw={hw} x{scale:g}", W, Wr, Wb)
    _check(f"attention_map hw={hw} x{scale:g}", out, outr, outb)


def test_attention_rejections(dev):
    """Shapes beyond the 220 KB tile (hw 6913..6976) and mismatched operands are refused before any launch."""
    lib = _lib.load()
    mk = torch.zeros(6976, 128, device=dev)
    pos = torch.zeros(1, 1, 64 * 16, 109 * 16, device=dev)
    small = torch.zeros(63, 128, device=dev)
    before = int(lib.mivos_launch_count())
    with pytest.raises(_lib.MivosError, match="attention_map"):
        ops.attention_map(mk, mk, 64, 109, pos, pos)
    for hw in (6913, 6976):
        with pytest.raises(_lib.MivosError, match="attention_weights"):
            ops.attention_weights(mk[:hw], mk[:hw])
    p7 = torch.zeros(1, 1, 7 * 16, 9 * 16, device=dev)
    for bad in (torch.zeros(1, 1, 7 * 16, 9 * 16 + 1, device=dev), torch.zeros(1, 2, 7 * 16, 9 * 16, device=dev),
                torch.zeros(7 * 16, 9 * 16, device=dev)):
        with pytest.raises(_lib.MivosError, match="pos/neg"):
            ops.attention_map(small, small, 7, 9, bad, p7)
        with pytest.raises(_lib.MivosError, match="pos/neg"):
            ops.attention_map(small, small, 7, 9, p7, bad)
    for a, b in ((small, small[:62]), (small, torch.zeros(63, 64, device=dev)), (torch.zeros(63, 64, device=dev),) * 2,
                 (small.reshape(1, 63, 128), small.reshape(1, 63, 128))):
        with pytest.raises(_lib.MivosError, match="attention_weights"):
            ops.attention_weights(a.contiguous(), b.contiguous())
    assert int(lib.mivos_launch_count()) == before


# ------------------------------------------------------------------------------------------------ aggregation


def _logits(groups, K, h4, w4, seed):
    """Object logits [groups*K, h4, w4]: random, +-30 (sigmoid rounds to 1.0 / saturates the clamp), exact zeros,
    and objects 1 tied with object 0 on a random subset of pixels."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(groups * K, h4, w4, generator=g) * 3
    pick = torch.randint(0, 4, base.shape, generator=g)
    lg = torch.where(pick == 0, torch.full_like(base, 30.0), torch.where(pick == 1, torch.full_like(base, -30.0),
                                                                         torch.where(pick == 2, torch.zeros_like(base), base)))
    lg = lg.reshape(groups, K, h4, w4)
    if K >= 2:
        tie = torch.rand(groups, h4, w4, generator=g) < 0.5
        lg[:, 1] = torch.where(tie, lg[:, 0], lg[:, 1])
    lg[0, :, 0, 0] = -30.0  # every object saturated low: bg = 1 in fp32
    return lg.reshape(groups * K, h4, w4)


@pytest.mark.parametrize("groups", [1, 3])
@pytest.mark.parametrize("K", [1, 2, 16])
def test_upsample4x_sigmoid_aggregate_ragged(dev, K, groups):
    for h4, w4 in ((1, 1), (3, 5), (7, 9)):
        H, W = 4 * h4, 4 * w4
        lg = _logits(groups, K, h4, w4, K * 100 + groups * 10 + h4).to(dev)
        cstride, coff = 7, 5  # the logits live in channel 5 of a 7-channel map: NaN in every other channel and the border
        halo = _halo(lg[:, None], cstride, coff, fill=NAN)
        raw = torch.full((groups * K, 1, H, W), SENT, device=dev)
        prob = torch.full(((groups,) if groups > 1 else ()) + (K + 1, 1, H, W), SENT, device=dev)
        ops.upsample4x_sigmoid_aggregate(halo, K, h4, w4, coff=coff, raw_out=raw, prob_out=prob, groups=groups)
        torch.cuda.synchronize()
        _lib.poll_kernel_error()
        tag = f"K={K} G={groups} {h4}x{w4}"
        # raw = sigmoid(bilinear x4): exact weights (multiples of 1/8), at most 4 roundings per corner term
        # (|dv| <= 4u B|l|, B = bilinear of |l|), carried by sigma' = p (1 - p); then 2 ulp of expf on exp(-v)
        # scaled by 1 - p, and one rounding each for 1 + t and the reciprocal
        v = _bilinear(lg[:, None], H, W)
        p = torch.sigmoid(v)
        rb = p * (1 - p) * 4 * U * _bilinear(lg.abs()[:, None], H, W) + p * (2 * U + 4 * U * (1 - p))
        _check(f"upsample4x raw {tag}", raw, p, rb)
        # prob: aggregation of the kernel's own fp32 raw, so a last-bit difference in p is not charged to it
        pr = raw.reshape(groups, K, H, W)
        pg = prob.reshape(groups, K + 1, H, W)
        for gi in range(groups):
            o, ob, _ = aggregate_reference(pr[gi])
            _check(f"upsample4x prob {tag} group {gi}", pg[gi], o, ob)
            _sum_and_range(f"upsample4x prob {tag} group {gi}", pg[gi], K)
        # aggregate_wbg on the same planes (the first group's)
        pk = raw[:K].contiguous()
        for keep_bg in (True, False):
            for const_bg in (False, True):
                got = ops.aggregate_wbg(pk, keep_bg=keep_bg, const_bg=const_bg)
                o, ob, _ = aggregate_reference(pk[:, 0], const_bg)
                what = f"aggregate_wbg {tag} keep_bg={keep_bg} const_bg={const_bg}"
                if keep_bg:
                    _check(what, got[:, 0], o, ob)
                    _sum_and_range(what, got[:, 0], K)
                else:
                    _check(what, got[:, 0], o[1:], ob[1:])
        for const_bg in (False, True):
            hard = ops.aggregate_wbg(pk, keep_bg=True, hard=True, const_bg=const_bg)[:, 0]
            _, _, lgt = aggregate_reference(pk[:, 0], const_bg)
            hl = 1000 * lgt
            top2 = hl.topk(2, 0).values
            clear = top2[0] - top2[1] > 20
            # where the fp64 hard-logit gap exceeds 20 the output is one-hot within K e^-19 (one unit of slack for the
            # kernel's own hard logits, 1000 x its logit error) plus the rounding of the sum
            onehot = F.one_hot(hl.argmax(0), K + 1).permute(2, 0, 1).double()
            tol = K * math.exp(-19) + (K + 1) * 2.0 ** -23
            dev_max = float(((hard.double() - onehot).abs().amax(0) * clear).max())
            print(f"aggregate_wbg hard {tag} const_bg={const_bg}: max one-hot deviation / bound = {dev_max / tol:.3g} "
                  f"on {int(clear.sum())} of {clear.numel()} pixels")
            assert dev_max <= tol, f"hard {tag}: one-hot deviation {dev_max:.3e} over {tol:.3e}"
            _sum_and_range(f"aggregate_wbg hard {tag} const_bg={const_bg}", hard, K)


def test_aggregate_rejects_17_objects(dev):
    lg = torch.zeros(17, 3, 3, 1, device=dev)
    with pytest.raises(_lib.MivosError, match="17 objects"):
        ops.upsample4x_sigmoid_aggregate(lg, 17, 1, 1)
    with pytest.raises(_lib.MivosError, match="17 objects"):
        ops.aggregate_wbg(torch.zeros(17, 1, 4, 4, device=dev))


# ------------------------------------------------------------------------------------------------ argmax, pad
PADS = [(0, 0, 0, 0), (3, 0, 0, 2), (0, 5, 1, 0), (1, 2, 3, 4)]  # (left, right, top, bottom)


@pytest.mark.parametrize("k1", [2, 17, 255])
def test_argmax_unpad_ragged(dev, k1):
    T, h, w = 3, 5, 7
    g = torch.Generator().manual_seed(k1)
    for pad in PADS:
        nh, nw = h + pad[2] + pad[3], w + pad[0] + pad[1]
        pr = torch.randint(0, 3, (k1, T, 1, nh, nw), generator=g).float() / 2  # three levels: many exact ties
        pr[-1, :, 0, 0, 0] = 2.0  # the last label wins a few pixels outright
        pr = pr.to(dev)
        ref = torch.argmax(pr.cpu(), 0).to(torch.uint8).to(dev)  # CPU argmax: the first maximum wins
        mp = torch.full((T, 1, nh, nw), 255, dtype=torch.uint8, device=dev)
        mo = torch.full((T, h, w), 255, dtype=torch.uint8, device=dev)
        ops.argmax_unpad(pr, pad, h, w, mp, mo)
        assert torch.equal(mp, ref), pad
        assert torch.equal(mo, ref[:, 0, pad[2]:pad[2] + h, pad[0]:pad[0] + w]), pad
        mp2 = torch.full_like(mp, 255)
        ops.argmax_unpad(pr, pad, h, w, mp2, None)
        assert torch.equal(mp2, ref), pad


def test_pad2d_ragged(dev):
    x = torch.randn(2, 3, 5, 7, device=dev)
    for pad in PADS:
        assert torch.equal(ops.pad2d(x, pad), F.pad(x, pad)), pad


# ------------------------------------------------------------------------------------------------ gathers, pooling
def _ragged_c(dtype):
    return (VEC[dtype], 40 if dtype == torch.float32 else 72)  # one vector, and a c that is not a multiple of 32


@pytest.mark.parametrize("dtype", [torch.float32, H16])
@pytest.mark.parametrize("h,w", [(2, 2), (6, 10), (34, 62)])
def test_maxpool_and_gather_s2_ragged(dev, dtype, h, w):
    n, ho, wo = 2, h // 2, w // 2
    g = torch.Generator().manual_seed(h * w)
    for c in _ragged_c(dtype):
        v = VEC[dtype]
        x = torch.randn(n, c, h, w, generator=g).relu().to(dtype).to(dev)  # post-ReLU, half the values exactly 0
        out = torch.full((n, ho + 2, wo + 2, c), SENT, dtype=dtype, device=dev)
        ops.maxpool3x3s2(_halo(x, c, dtype=dtype), n, h, w, out)
        exp = _halo(F.max_pool2d(x.double(), 3, 2, 1), c, fill=SENT, dtype=dtype)
        assert torch.equal(out, exp), f"maxpool c={c}"
        # gather_s2 from the first c channels of a wider map (sentinel in the others, zero border in the window)
        xw = torch.full((n, h + 2, w + 2, c + v), SENT, dtype=dtype, device=dev)
        xw[..., :c] = _halo(x, c, dtype=dtype)
        for ks in (1, 3):
            kk = ks * ks
            oc = kk * c + v  # pad columns past the taps keep the sentinel
            gm = torch.full((n, ho + 2, wo + 2, oc), SENT, dtype=dtype, device=dev)
            ops.gather_s2(xw, n, h, w, c, ks, gm)
            cols = F.unfold(x.double(), ks, padding=ks // 2, stride=2)  # [n, c*kk, ho*wo], (c, ky, kx) order
            cols = cols.reshape(n, c, kk, ho, wo).permute(0, 3, 4, 2, 1).reshape(n, ho, wo, kk * c)
            exp = torch.full_like(gm, SENT)
            exp[..., :kk * c] = 0  # HALO rows of the matrix are zero rows
            exp[:, 1:-1, 1:-1, :kk * c] = cols.to(dtype)
            assert torch.equal(gm, exp), f"gather_s2 ks={ks} c={c}"


@pytest.mark.parametrize("dtype", [torch.float32, H16])
@pytest.mark.parametrize("h,w", [(2, 2), (6, 10), (34, 62)])
def test_upsample2x_add_ragged(dev, dtype, h, w):
    n, hs, ws = 2, h // 2, w // 2
    g = torch.Generator().manual_seed(h * w + 1)
    for c in _ragged_c(dtype):
        for mode in ("add", "relu", "skip1", "skip2"):
            x = torch.randn(n, c, h, w, generator=g).to(dtype).to(dev)
            u = torch.randn(n, c, hs, ws, generator=g).to(dtype).to(dev)
            xh = _halo(x, c, fill=SENT, dtype=dtype)
            uh = _halo(u, c, fill=NAN, dtype=dtype)  # the bilinear source's border is never read
            xr = torch.full_like(xh, SENT) if mode == "relu" else None
            skip = base = None
            if mode.startswith("skip"):
                s_n = int(mode[-1])
                sk = torch.randn(s_n, c, h, w, generator=g).to(dtype).to(dev)
                skip = _halo(sk, c, fill=NAN, dtype=dtype)
                base = sk.repeat_interleave(n // s_n, 0)  # skip map j serves images [j n/S, (j+1) n/S)
            else:
                base = x
            ops.upsample2x_add(xh, uh, n, h, w, x_relu=xr, skip=skip)
            torch.cuda.synchronize()
            ref = base.double() + _bilinear(u, h, w)
            # exact weights (multiples of 1/16); each corner term passes at most 5 roundings (two products, two
            # sums, the addition of x): 5u (|x| + sum |w v|); fp16 maps round the result once more (2^-11 |ref|,
            # 2^-25 absolute below the normal range)
            mag = base.double().abs() + _bilinear(u.abs(), h, w)
            bound = 5 * U * mag
            if dtype == H16:
                bound = bound * (1 + 2.0 ** -11) + 2.0 ** -11 * ref.abs() + 2.0 ** -25
            _check(f"upsample2x_add {dtype} {h}x{w} c={c} {mode}", xh[:, 1:-1, 1:-1].permute(0, 3, 1, 2), ref, bound)
            assert bool((xh[:, 0] == SENT).all() and (xh[:, -1] == SENT).all() and (xh[:, :, 0] == SENT).all()
                        and (xh[:, :, -1] == SENT).all()), "HALO border of x written"
            if xr is not None:
                assert torch.equal(xr[:, 1:-1, 1:-1], xh[:, 1:-1, 1:-1].relu())
                inner = torch.zeros_like(xr, dtype=torch.bool)
                inner[:, 1:-1, 1:-1] = True
                assert bool((xr[~inner] == SENT).all()), "HALO border of x_relu written"


# ------------------------------------------------------------------------------------------------ layout copies
@pytest.mark.parametrize("dtype", [torch.float32, H16])
@pytest.mark.parametrize("c", [1, 33, 100])
def test_halo_nchw_transposes_ragged(dev, dtype, c):
    n, coff = 2, 3
    cs = coff + c + 2
    g = torch.Generator().manual_seed(c)
    for h, w in ((5, 7), (9, 13)):  # 35 and 117 pixels: ragged 32-pixel tiles; c = 33, 100: ragged channel tiles
        x = torch.randn(n, c, h, w, generator=g).to(dev)
        for relu in (False, True):
            hb = torch.full((n, h + 2, w + 2, cs), SENT, dtype=dtype, device=dev)
            ops.nchw_to_halo(x, hb, coff=coff, relu=relu)
            exp = _halo(x.relu() if relu else x, cs, coff, fill=SENT, dtype=dtype)
            assert torch.equal(hb, exp), f"nchw_to_halo {h}x{w} relu={relu}"
        src = torch.randn(n, h + 2, w + 2, cs, generator=g).to(dtype).to(dev)  # border and other channels: noise
        out = torch.full((n, c, h, w), SENT, device=dev)
        ops.halo_to_nchw(src, n, h, w, c, coff, out=out)
        assert torch.equal(out, src[:, 1:-1, 1:-1, coff:coff + c].permute(0, 3, 1, 2).float()), f"halo_to_nchw {h}x{w}"


def test_halo_to_pixels_ragged(dev):
    n, h, w, cs = 2, 5, 7, 24
    src = torch.randn(n, h + 2, w + 2, cs, device=dev)
    for coff, c in ((4, 12), (8, 16), (0, 24)):
        out = torch.full((n * h * w + 1, c), SENT, device=dev)  # one row past the end must survive
        ops.halo_to_pixels(src, n, h, w, coff, c, out)
        assert torch.equal(out[:-1], src[:, 1:-1, 1:-1, coff:coff + c].reshape(n * h * w, c)), (coff, c)
        assert bool((out[-1] == SENT).all())


@pytest.mark.parametrize("src_dtype,dst_dtype", [(torch.float32, torch.float32), (torch.float32, H16),
                                                 (H16, torch.float32), (H16, H16)])
def test_halo_copy_ragged(dev, src_dtype, dst_dtype):
    n, h, w, c = 3, 5, 7, 12
    g = torch.Generator().manual_seed(5)
    for src_n in (1, 3):  # 1: one map broadcast over the n images
        for relu in (False, True):
            src = torch.randn(src_n, h + 2, w + 2, 17, generator=g).to(src_dtype).to(dev)
            dst = torch.full((n, h + 2, w + 2, 21), SENT, dtype=dst_dtype, device=dev)
            ops.halo_copy(src, dst, n, h, w, c, src_coff=3, dst_coff=5, relu=relu)  # odd channel offsets
            v = src[:, 1:-1, 1:-1, 3:3 + c].float()
            v = (v.relu() if relu else v).repeat_interleave(n // src_n, 0)
            exp = torch.full_like(dst, SENT)
            exp[:, 1:-1, 1:-1, 5:5 + c] = v.to(dst_dtype)
            assert torch.equal(dst, exp), (src_n, relu)


def test_bank_write_ragged(dev):
    """K = 3 objects of 5 x 7 pixels; keys from channels [520, 648), values from [4, 516) of a 652-channel map.
    Slot t = 2 is the last one ((t+1) hw = capacity).  The device-scalar form must match the static one bit for bit."""
    K, h, w, T = 3, 5, 7, 3
    hw, cap, cs, ck, cv = 35, 3 * 35, 652, 520, 4
    g = torch.Generator().manual_seed(9)
    halo = torch.randn(K, h + 2, w + 2, cs, generator=g).to(dev)
    keys = halo[:, 1:-1, 1:-1, ck:ck + 128].reshape(K, hw, 128)
    vals = halo[:, 1:-1, 1:-1, cv:cv + 512].reshape(K, hw, 512)
    dyn_t = torch.zeros(1, dtype=torch.int32, device=dev)
    for t in (0, 2):
        banks = []
        for dyn in (False, True):
            bk = torch.full((K, cap, 128), SENT, device=dev)
            bv = torch.full((K, cap, 512), SENT, device=dev)
            if dyn:
                ops.store_i32(dyn_t, t)
                ops.bank_write(halo, K, h, w, ck, cv, bk, bv, T - 1, dyn_t=dyn_t)  # T - 1: the largest slot it may name
            else:
                ops.bank_write(halo, K, h, w, ck, cv, bk, bv, t)
            banks.append((bk, bv))
        ek = torch.full((K, cap, 128), SENT, device=dev)
        ev = torch.full((K, cap, 512), SENT, device=dev)
        ek[:, t * hw:(t + 1) * hw] = keys
        ev[:, t * hw:(t + 1) * hw] = vals
        assert torch.equal(banks[0][0], ek) and torch.equal(banks[0][1], ev), t
        assert torch.equal(banks[1][0], banks[0][0]) and torch.equal(banks[1][1], banks[0][1]), t
    with pytest.raises(_lib.MivosError):
        ops.bank_write(halo, K, h, w, ck, cv, bk, bv, T)  # one slot past the capacity


def test_bank_from_nchw_ragged(dev):
    K, T, h, w, cap = 2, 2, 5, 7, 100  # 70 slots: not a multiple of 32, below the capacity
    g = torch.Generator().manual_seed(13)
    keys = torch.randn(K, 128, T, h, w, generator=g).to(dev)
    vals = torch.randn(K, 512, T, h, w, generator=g).to(dev)
    bk = torch.full((K, cap, 128), SENT, device=dev)
    bv = torch.full((K, cap, 512), SENT, device=dev)
    ops.bank_from_nchw(keys, vals, bk, bv)
    slots = T * h * w
    ek, ev = torch.full_like(bk, SENT), torch.full_like(bv, SENT)
    ek[:, :slots] = keys.permute(0, 2, 3, 4, 1).reshape(K, slots, 128)
    ev[:, :slots] = vals.permute(0, 2, 3, 4, 1).reshape(K, slots, 512)
    assert torch.equal(bk, ek) and torch.equal(bv, ev)


@pytest.mark.parametrize("dtype", [torch.float32, H16])
@pytest.mark.parametrize("cpad", [16, 32])
def test_fusion_gather_ragged(dev, dtype, cpad):
    h, w = 7, 9
    g = torch.Generator().manual_seed(cpad)
    im = torch.randn(1, 3, h, w, generator=g).to(dev)
    seg1, seg2 = torch.rand(1, 1, h, w, generator=g).to(dev), torch.rand(1, 1, h, w, generator=g).to(dev)
    attn = torch.rand(1, 2, h, w, generator=g).to(dev)
    nc, nr = 0.3, 0.7
    out = torch.full((1, h + 2, w + 2, cpad), SENT, dtype=dtype, device=dev)
    ops.fusion_gather(im, seg1, seg2, attn, nc, nr, out)
    planes = torch.cat([im, seg1, seg2, attn, torch.full((1, 1, h, w), nc, device=dev),
                        torch.full((1, 1, h, w), nr, device=dev)], 1)  # fp32 constants, as the ABI passes them
    exp = _halo(planes, cpad, fill=0.0, border=SENT, dtype=dtype)  # channels 9..cpad are zero
    assert torch.equal(out, exp)


def test_halo_sigmoid_to_plane_ragged(dev):
    h, w, cs, coff = 7, 9, 6, 5
    g = torch.Generator().manual_seed(17)
    lg = torch.linspace(-80, 80, h * w).reshape(1, 1, h, w)
    lg = lg + torch.randn(1, 1, h, w, generator=g).clamp(-0.5, 0.5) * (lg.abs() < 79)
    lg = lg.to(dev)
    halo = _halo(lg, cs, coff, fill=NAN)
    plane = torch.full((h * w + 1,), SENT, device=dev)  # one element past the plane must survive
    ops.halo_sigmoid_to_plane(halo, h, w, coff, plane)
    torch.cuda.synchronize()
    ref = torch.sigmoid(lg.double()).reshape(-1)
    # 1 / (1 + expf(-x)): 2 ulp of expf scaled by 1 - sigma, one rounding each for the sum and the reciprocal
    # (at most 6u relative: within 4 to 6 ulp of the fp32 result)
    _check("halo_sigmoid_to_plane", plane[:-1], ref, ref * (2 * U + 4 * U * (1 - ref)))
    assert float(plane[-1]) == SENT


# ------------------------------------------------------------------------------------------------ stem gathers
def _stem_out(N, H, W, kpad, dtype, dev):
    """A matrix of N * (H/2 + 2) * (W/2 + 2) rows filled with the sentinel, plus one guard row past its end."""
    rows = N * (H // 2 + 2) * (W // 2 + 2)
    buf = torch.full((rows + 1, kpad), SENT, dtype=dtype, device=dev)
    return buf, buf[:rows]


def _check_stem(what, buf, img, bound, kpad, s2d, dtype):
    """Channels other than "others": bit-exact after one rounding to the map type.  "others" (channel 4 of the mask
    form, K >= 3): within its bound, exact where that is 0 (zero padding).  Guard row untouched."""
    cin = img.shape[1]
    assert bool((buf[-1] == SENT).all()), f"{what}: wrote past the matrix"
    got = buf[:-1].double()
    rounded = img.to(dtype).double()
    if bound.any():  # the "others" channel keeps its exact sum, the other channels their rounded value
        rounded[:, 4] = img[:, 4]
    ref = stem_matrix(rounded, kpad, s2d)
    if not bound.any():
        assert torch.equal(got, ref), what
        return
    bnd = _round16(stem_matrix(bound, kpad, s2d), ref, dtype)
    col = torch.arange(kpad, device=buf.device)
    oc = (col < (16 if s2d else 49) * cin) & (col % cin == 4)
    assert torch.equal(got[:, ~oc], ref[:, ~oc]), f"{what}: frame / own-mask / pad columns"
    go, ro, bo = got[:, oc], ref[:, oc], bnd[:, oc]
    live = (ro != 0) | (bo != 0)
    assert torch.equal(go[~live], ro[~live]), f"{what}: others in the zero padding"
    _check(f"{what} others", go[live], ro[live], bo[live])


@pytest.mark.parametrize("dtype", [torch.float32, H16])
@pytest.mark.parametrize("s2d", [False, True])
@pytest.mark.parametrize("K", [1, 2, 16])
def test_stem_gather_masks_ragged(dev, dtype, s2d, K):
    """The memorize stem: frame + K masks -> per object (frame, own mask, others).  One group at h = 2 (a single
    output row), w = 2 and a ragged 14 x 22; three groups whose frames and masks lie frame_gstride / mask_gstride
    apart with NaN in the gaps between the clips."""
    kpad = 96 if s2d else 256  # 16 * 5 = 80 / 49 * 5 = 245 gathered columns: the rest must be written as zeros
    fn = _lib.lib().mivos_stem_gather_s2d if s2d else _lib.lib().mivos_stem_gather
    g = torch.Generator().manual_seed(K * 10 + int(s2d))
    for G, H, W in ((1, 2, 10), (1, 6, 2), (1, 14, 22), (3, 6, 10)):
        hw = H * W
        frames = torch.randn(G, 3, H, W, generator=g)
        masks = torch.rand(G, K, H, W, generator=g)
        fgs, mgs = (3 * hw + hw + 7, K * hw + hw + 5) if G > 1 else (0, 0)
        fbuf = torch.full((max(G * fgs, 3 * hw),), NAN)
        mbuf = torch.full((max(G * mgs, K * hw),), NAN)
        for gi in range(G):
            fbuf[gi * fgs:gi * fgs + 3 * hw] = frames[gi].reshape(-1)
            mbuf[gi * mgs:gi * mgs + K * hw] = masks[gi].reshape(-1)
        fbuf, mbuf = fbuf.to(dev), mbuf.to(dev)
        buf, out = _stem_out(G * K, H, W, kpad, dtype, dev)
        _lib.check(fn(ops._ptr(fbuf), ops._ptr(mbuf), K, H, W, ops._ptr(out), kpad, ops._f16(out), G, fgs, mgs,
                      ops._stream()), "stem_gather")
        torch.cuda.synchronize()
        _lib.poll_kernel_error()
        img, bound = stem_images(frames.to(dev), masks.to(dev))
        _check_stem(f"stem_gather s2d={s2d} {dtype} K={K} G={G} {H}x{W}", buf, img, bound, kpad, s2d, dtype)
        if G == 1:  # the wrapper's [K, 1, H, W] form is the same launch
            buf2, out2 = _stem_out(K, H, W, kpad, dtype, dev)
            ops.stem_gather(frames.to(dev), masks[0, :, None].contiguous().to(dev), out2, s2d=s2d)
            assert torch.equal(buf2, buf)


@pytest.mark.parametrize("dtype", [torch.float32, H16])
def test_stem_gather_frames_ragged(dev, dtype):
    """Batches of frames: cin 3 through mivos_stem_gather (49 taps and s2d) and mivos_stem_gather_frames, cin 6 (the
    S2M stem: image, previous mask, +/- scribbles) through mivos_stem_gather_frames; h = 2, w = 2, ragged, and the
    widest 6-channel frame the shared-memory check admits, 1376 pixels in fp32 (7 rows x 1382 x 6 x 4 B = 232344 B
    of the 232448) and 2760 in fp16."""
    g = torch.Generator().manual_seed(6)
    widest = 1376 if dtype == torch.float32 else 2760
    for cin in (3, 6):
        for n, H, W in ((2, 2, 2), (2, 2, 14), (2, 10, 2), (2, 6, 22)) + (((1, 2, widest),) if cin == 6 else ()):
            frames = torch.randn(n, cin, H, W, generator=g).to(dev)
            img, bound = stem_images(frames)
            kpad = 160 if cin == 3 else 320
            buf, out = _stem_out(n, H, W, kpad, dtype, dev)
            ops.stem_gather_frames(frames, out)
            torch.cuda.synchronize()
            _lib.poll_kernel_error()
            _check_stem(f"stem_gather_frames cin={cin} {dtype} n={n} {H}x{W}", buf, img, bound, kpad, False, dtype)
            if cin == 3:
                for s2d, kp in ((False, kpad), (True, 56)):
                    buf, out = _stem_out(n, H, W, kp, dtype, dev)
                    ops.stem_gather(frames, None, out, s2d=s2d)
                    torch.cuda.synchronize()
                    _check_stem(f"stem_gather s2d={s2d} cin=3 {dtype} n={n} {H}x{W}", buf, img, bound, kp, s2d, dtype)


# ------------------------------------------------------------------------------------------------ graph staging
# Every replayed frame depends on these (inference_core.py, lockstep.py): the int32 bank counters, the pointer table
# of the frame, and the copies that stage its operands and deliver its result planes.  All bit-exact, with sentinels
# on both sides of every destination.
I32_SENT, I64_SENT, BSENT = -7, -0x0123456789ABCDEF, 0xA5
GUARD = 256  # sentinel bytes on each side of a copy destination (keeps the payload 16-byte aligned)


def test_store_i32_ragged(dev):
    vals = [2 ** 31 - 1, -2 ** 31, 0, 12345]
    buf = torch.empty(8, dtype=torch.int32, device=dev)
    for n in range(1, 5):
        buf.fill_(I32_SENT)
        ops.store_i32(buf[2:], *vals[:n])
        exp = torch.full((8,), I32_SENT, dtype=torch.int32)
        exp[2:2 + n] = torch.tensor(vals[:n], dtype=torch.int32)
        assert torch.equal(buf.cpu(), exp), n


def test_store_words_ragged(dev):
    """n64 = 0, 1, 37, 64 words with n32 = 0..4 counters; 130 words take three launches of the wrapper (64 + 64 + 2),
    the counters going with the first."""
    import random
    rnd = random.Random(5)
    b64 = torch.empty(134, dtype=torch.int64, device=dev)
    b32 = torch.empty(8, dtype=torch.int32, device=dev)
    for n64, n32s in ((0, range(5)), (1, range(5)), (37, range(5)), (64, range(5)), (130, (0, 4))):
        for n32 in n32s:
            w64 = [rnd.getrandbits(64) - 2 ** 63 for _ in range(n64)]
            w32 = [rnd.getrandbits(32) - 2 ** 31 for _ in range(n32)]
            b64.fill_(I64_SENT), b32.fill_(I32_SENT)
            ops.store_words(b64[2:], w64, b32[2:], w32)
            e64 = torch.full((134,), I64_SENT, dtype=torch.int64)
            e64[2:2 + n64] = torch.tensor(w64, dtype=torch.int64)
            e32 = torch.full((8,), I32_SENT, dtype=torch.int32)
            e32[2:2 + n32] = torch.tensor(w32, dtype=torch.int32)
            assert torch.equal(b64.cpu(), e64) and torch.equal(b32.cpu(), e32), (n64, n32)


def _guarded(nbytes, dev):
    """(buffer, payload): nbytes payload bytes between GUARD sentinel bytes on each side, inside one allocation."""
    buf = torch.full((nbytes + 2 * GUARD,), BSENT, dtype=torch.uint8, device=dev)
    return buf, buf[GUARD:GUARD + nbytes]


def _i64(vals, dev):
    return torch.tensor(vals, dtype=torch.int64, device=dev)


@pytest.mark.parametrize("dyn_is_src", [True, False])
def test_copy_segments_ragged(dev, dyn_is_src):
    """Segments of 16 B, 4 KB + 16 B, 20 MB (longer than one grid-stride sweep, about 8.6 MB on 132 SMs) and two
    other sizes, all different and below max_bytes; a sixth segment has dyn = 0 and must copy nothing, in particular
    not onto its fixed side."""
    sizes = [16, 4096 + 16, 20 << 20, 160, 65536 + 48, 4096]
    skip = len(sizes) - 1
    gen = torch.Generator(device=dev).manual_seed(7)
    srcs = [torch.randint(0, 256, (s,), dtype=torch.uint8, device=dev, generator=gen) for s in sizes]
    dsts = [_guarded(s, dev) for s in sizes]
    src_p = [s.data_ptr() for s in srcs]
    dst_p = [p.data_ptr() for _, p in dsts]
    fixed, dyn = (dst_p, src_p) if dyn_is_src else (src_p, dst_p)
    dyn = [0 if i == skip else p for i, p in enumerate(dyn)]
    ops.copy_segments(_i64(fixed, dev), _i64(dyn, dev), _i64(sizes, dev), len(sizes), dyn_is_src, (20 << 20) + 4096)
    torch.cuda.synchronize()
    _lib.poll_kernel_error()
    for i, (buf, payload) in enumerate(dsts):
        g0, g1 = buf[:GUARD], buf[GUARD + sizes[i]:]
        assert bool((g0 == BSENT).all() and (g1 == BSENT).all()), f"segment {i} ({sizes[i]} B) overran its destination"
        if i == skip:
            assert bool((payload == BSENT).all()), "a skipped segment wrote its destination"
        else:
            assert torch.equal(payload, srcs[i]), f"segment {i} ({sizes[i]} B)"


def test_copy_segments_graph_replay(dev):
    """A frame step as inference_core.py records it: ONE captured graph stages three segments into fixed buffers
    (dyn sources) and delivers them again (dyn destinations); between replays store_words rewrites the pointer table.
    The third replay skips segment 1 both ways (pointer 0): its staging buffer keeps the previous frame's bytes."""
    sizes = [16, 4096 + 16, 1 << 20]
    n = len(sizes)
    gen = torch.Generator(device=dev).manual_seed(8)
    stage = [_guarded(s, dev) for s in sizes]
    fixed = _i64([p.data_ptr() for _, p in stage], dev)
    nbytes = _i64(sizes, dev)
    table = torch.zeros(2 * n, dtype=torch.int64, device=dev)  # [sources..., destinations...]
    frames = [([torch.randint(0, 256, (s,), dtype=torch.uint8, device=dev, generator=gen) for s in sizes],
               [_guarded(s, dev) for s in sizes]) for _ in range(4)]

    def step(f, skip=None):
        srcs, dsts = frames[f]
        ptrs = [0 if i == skip else s.data_ptr() for i, s in enumerate(srcs)]
        ptrs += [0 if i == skip else p.data_ptr() for i, (_, p) in enumerate(dsts)]
        ops.store_words(table, ptrs)

    def body():
        ops.copy_segments(fixed, table[:n], nbytes, n, True, max(sizes))
        ops.copy_segments(fixed, table[n:], nbytes, n, False, max(sizes))

    def check(f, skip=None, kept=None):
        torch.cuda.synchronize()
        _lib.poll_kernel_error()
        srcs, dsts = frames[f]
        for i in range(n):
            want = kept if i == skip else srcs[i]
            for buf, payload, sent in ((*stage[i], want), (*dsts[i], None if i == skip else srcs[i])):
                assert bool((buf[:GUARD] == BSENT).all() and (buf[GUARD + sizes[i]:] == BSENT).all()), (f, i)
                assert bool((payload == BSENT).all()) if sent is None else torch.equal(payload, sent), (f, i)

    step(0)
    body()  # eagerly once, as InferenceCore does before capturing
    check(0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()
    for f, skip in ((1, None), (2, 1), (3, None)):
        step(f, skip)
        graph.replay()
        check(f, skip, kept=frames[f - 1][0][1])
