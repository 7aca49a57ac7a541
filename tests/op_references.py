"""TEST INFRASTRUCTURE: float64 references of the non-GEMM operators and the elementwise bounds derived for them, in
one place for the ragged-shape tests (tests/test_gpu_ops_ragged.py, test_gpu_hires_ops.py, test_gpu_z_s2m.py,
test_gpu_many_objects.py) and the operator census (tests/op_census.py).  Each reference is computed from the operands
the kernel saw; each bound is written as a formula with its derivation.  Device-agnostic and importable without a
GPU."""
import math

import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24  # unit roundoff of fp32 (round to nearest)
H16 = torch.float16


def _bilinear(x, h, w):
    """fp64 bilinear resize, align_corners=False (the kernels' source-index convention)."""
    return F.interpolate(x.double(), size=(h, w), mode="bilinear", align_corners=False)


def round16(bound, ref, dtype):
    """A bound on an fp32 value, widened by its final rounding to an fp16 map (2^-25 absolute below the normal range)."""
    if dtype != H16:
        return bound
    return bound * (1 + 2.0 ** -11) + 2.0 ** -11 * ref.abs() + 2.0 ** -25


# ------------------------------------------------------------------------------------------------ attention
# Logit s_ij = sum_c mk_ic * fl(qk_jc / fl(sqrt 128)): the fp32 constant and the division round once each, the
# 128-term fma chain rounds 128 times, so |s_ij - L_ij| <= GAMMA * S_ij with S_ij = sum_c |mk_ic qk_jc| / sqrt(128).
GAMMA = 130 * U


def attention_reference(mk, qk, h16=None, w16=None, pos=None, neg=None):
    """fp64 W[i, j] = softmax_i(mk_i . qk_j / sqrt(128)) with its elementwise bound; with pos/neg also the map
    bilinear_x16(area16(pos|neg) @ W) and its bound."""
    hw = mk.shape[0]
    m, q = mk.double(), qk.double()
    L = m @ q.t() / math.sqrt(128)  # [memory i, query j]
    S = m.abs() @ q.abs().t() / math.sqrt(128)
    Lmax = L.max(0, keepdim=True).values
    W = torch.softmax(L, 0)
    # relative error of e_ij = expf(fl(s_ij - m_j)): the logit and the column max (|m_j - Lmax_j| <= GAMMA max_i S_ij),
    # one rounding of the difference (u |L_ij - Lmax_j|), 2 ulp of expf (4u)
    eps = GAMMA * (S + S.max(0, keepdim=True).values) + U * (L - Lmax).abs() + 4 * U
    del S
    # den_j = sum_i e_ij: ceil(hw/32) additions per lane + 5 levels of the warp tree, +1 for gamma_n ~ n u
    g_den = (math.ceil(hw / 32) + 6) * U
    d_den = (W * eps).sum(0, keepdim=True) + g_den  # relative error of den_j: the e_ij errors weighted by W_ij
    # W_ij = fl(e_ij / den_j): + one rounding; expf and the quotient lose relative precision below 2^-126, where
    # their absolute error stays within 4 * 2^-149
    Wb = W * (eps + d_den + U) + 4 * 2.0 ** -149
    if pos is None:
        return W, Wb
    pooled = torch.cat([F.avg_pool2d(pos.double(), 16), F.avg_pool2d(neg.double(), 16)], 1).reshape(2, hw)
    mp = pooled @ W  # [2, hw]
    # map_j = pp_j / den_j is the W-weighted mean of pooled, so to first order the e_ij errors enter only as
    # sum_i W_ij eps_ij |pooled_i - map_j| (an error common to all e_ij cancels).  pooled_i >= 0 is 255 sequential
    # fp32 additions (the /256 is exact): 255u of it, i.e. 255u map_j after weighting; pp_j and den_j round g_den
    # each; the quotient rounds once
    We = W * eps
    del eps
    mb = torch.stack([(We * (pooled[k][:, None] - mp[k][None, :]).abs()).sum(0) for k in range(2)])
    mb = mb + mp * (255 * U + 2 * g_den + U)
    del We
    H, Wd = 16 * h16, 16 * w16
    out = _bilinear(mp.reshape(1, 2, h16, w16), H, Wd)
    # x16 bilinear: exact weights (multiples of 1/32), at most 4 roundings on each corner term, and nonnegative
    # weights carry the map bound through
    outb = _bilinear(mb.reshape(1, 2, h16, w16), H, Wd) + 4 * U * _bilinear(mp.abs().reshape(1, 2, h16, w16), H, Wd)
    return W, Wb, out, outb


# Streamed attention (attention_stream_kernel): keys in tiles of SK, a running maximum and rescales; the bound is
# derived in the docstring of tests/test_gpu_hires_ops.py (DESIGN.md section 6).
SK = 128  # keys per tile of attention_stream_kernel
TINY = 2.0 ** -149
BLOCK = 1024  # query columns per float64 block


def _tiles(x, fill):
    """[hw, nb] -> [T, SK, nb] padded with `fill`."""
    hw, nb = x.shape
    T = -(-hw // SK)
    p = torch.full((T * SK, nb), fill, dtype=x.dtype, device=x.device)
    p[:hw] = x
    return p.reshape(T, SK, nb)


def stream_blocks(mk, qk, pooled=None, row_lse=None):
    """Yields, per block of query columns [j0, j1): float64 logits and softmax W over the memory axis, the streamed
    kernel's per-term relative error eps (with rescales) and the resident kernel's eps_r; with pooled also the map,
    and with row_lse (logsumexp over queries of every memory row) the map of a softmax over the QUERY axis."""
    hw = mk.shape[0]
    m, q = mk.double(), qk.double()
    for j0 in range(0, hw, BLOCK):
        j1 = min(hw, j0 + BLOCK)
        L = m @ q[j0:j1].t() / math.sqrt(128)
        S = m.abs() @ q[j0:j1].abs().t() / math.sqrt(128)
        Lmax = L.max(0, keepdim=True).values
        W = torch.softmax(L, 0)
        G = GAMMA * _tiles(S, 0.0).max(1).values  # [T, nb]: |fp32 tile max - float64 tile max| <= G
        tmax = _tiles(L, -math.inf).max(1).values
        lo = torch.cummax(tmax - G, 0).values
        possible = torch.zeros_like(tmax)
        possible[1:] = ((tmax[1:] + G[1:]) > lo[:-1]).double()
        after = possible.flip(0).cumsum(0).flip(0) - possible  # rescales strictly after tile t
        R = after.repeat_interleave(SK, 0)[:hw]
        base = GAMMA * (S + S.max(0, keepdim=True).values)
        dl = (L - Lmax).abs()
        del S
        eps = base + 2 * U * dl + 4 * U * (1 + R)
        eps_r = base + U * dl + 4 * U
        blk = dict(j0=j0, j1=j1, L=L, W=W, eps=eps, eps_r=eps_r, tmax=tmax)
        if pooled is not None:
            blk["map"] = pooled @ W
        if row_lse is not None:
            blk["map_qaxis"] = pooled @ torch.exp(L - row_lse[:, None])
        yield blk


def weights_streamed_blocks(mk, qk):
    """Yields (j0, j1, W, bound) of attention_weights_streamed per block of query columns: W's second pass uses the
    final maximum, so its exponentials carry the resident kernel's eps_r, and only the denominator carries the
    streamed errors ((5T + 6)u of the lane partials plus hw TINY of flushed terms)."""
    hw = mk.shape[0]
    g_s = (5 * (-(-hw // SK)) + 6) * U
    for b in stream_blocks(mk, qk):
        W = b["W"]
        d_den = (W * b["eps"]).sum(0, keepdim=True) + g_s + hw * TINY
        yield b["j0"], b["j1"], W, W * (b["eps_r"] + d_den + U) + 4 * TINY


def map_reference(mk, qk, h16, w16, pos, neg, mistakes=False):
    """float64 map [1,2,H,W], the streamed bound, the resident bound (same formula as attention_reference), and with
    `mistakes` the maps of three kernel mistakes: the last tile skipped, no rescale, the softmax over queries."""
    hw = h16 * w16
    T = -(-hw // SK)
    pooled = torch.cat([F.avg_pool2d(pos.double(), 16), F.avg_pool2d(neg.double(), 16)], 1).reshape(2, hw)
    row_lse = None
    if mistakes:
        m, q = mk.double(), qk.double()
        row_lse = torch.full((hw,), -math.inf, dtype=torch.float64, device=mk.device)
        for j0 in range(0, hw, BLOCK):
            row_lse = torch.logaddexp(row_lse, torch.logsumexp(m @ q[j0:j0 + BLOCK].t() / math.sqrt(128), 1))
    g_s = (5 * T + 6) * U
    g_r = (math.ceil(hw / 32) + 6) * U
    mp = torch.empty(2, hw, dtype=torch.float64, device=mk.device)
    mb, mbr = torch.empty_like(mp), torch.empty_like(mp)
    bad = {k: torch.empty_like(mp) for k in ("skip_last_tile", "no_rescale", "query_axis")} if mistakes else {}
    for b in stream_blocks(mk, qk, pooled, row_lse):
        j0, j1, W, mapb = b["j0"], b["j1"], b["W"], b["map"]
        mp[:, j0:j1] = mapb
        for k in range(2):
            dev_ = (pooled[k][:, None] - mapb[k][None, :]).abs()
            mb[k, j0:j1] = (W * b["eps"] * dev_).sum(0)
            mbr[k, j0:j1] = (W * b["eps_r"] * dev_).sum(0)
        if mistakes:
            L = b["L"]
            cut = (T - 1) * SK
            bad["skip_last_tile"][:, j0:j1] = pooled[:, :cut] @ torch.softmax(L[:cut], 0)
            run = torch.cummax(b["tmax"], 0).values.repeat_interleave(SK, 0)[:hw]  # running max after each key's tile
            e = torch.exp(L - run)
            bad["no_rescale"][:, j0:j1] = (pooled @ e) / e.sum(0)
            bad["query_axis"][:, j0:j1] = b["map_qaxis"]
    mb = mb + mp * (255 * U + 2 * g_s + U) + 2 * hw * TINY
    mbr = mbr + mp * (255 * U + 2 * g_r + U)
    H, Wd = 16 * h16, 16 * w16
    up = lambda x: F.interpolate(x.reshape(1, 2, h16, w16), size=(H, Wd), mode="bilinear", align_corners=False)  # noqa: E731
    out = up(mp)
    lift = 4 * U * up(mp.abs())
    return out, up(mb) + lift, up(mbr) + lift, {k: up(v) for k, v in bad.items()}


# ------------------------------------------------------------------------------------------------ aggregation
CLAMP_LO = float(np.float32(1e-7))  # the kernel's fp32 clamp bounds, not the decimal constants
CLAMP_HI = float(np.float32(1.0) - np.float32(1e-7))
assert CLAMP_HI == 1.0 - 2.0 ** -23


def aggregate_reference(p, const_bg=False):
    """fp64 aggregate_wbg of the fp32 object probabilities p [K, ...] (the kernel's operands, exactly):
    softmax over [bg, p_1..p_K] of logit(clamp(.)), with bg = prod(1 - p) (0.5 for const_bg); and its bound."""
    K = p.shape[0]
    v = p.double()
    bg = torch.full_like(v[:1], 0.5) if const_bg else torch.prod(1 - v, 0, keepdim=True)
    x = torch.cat([bg, v], 0).clamp(CLAMP_LO, CLAMP_HI)
    lg = torch.log(x / (1 - x))
    o = torch.softmax(lg, 0)
    # relative error of the fp32 operand: bg is K roundings of 1 - p_j and K - 1 of the product; p_j are exact
    rho = torch.zeros_like(x)
    if not const_bg:
        rho[0] = 2 * K * U
    # absolute error of each fp32 logit: the operand's error through d logit / dx = 1 / (x (1 - x)), one rounding
    # each for 1 - x and the quotient, 1 ulp of logf (<= 2u |logit|)
    eta = rho / (1 - x) + 2 * U + 2 * U * lg.abs()
    # relative error of e_j = expf(fl(l_j - max)): eta_j, the rounded difference, 2 ulp of expf.  o_j = e_j / s:
    # s carries the e errors weighted by o plus K additions, and the quotient rounds once
    a = eta + U * (lg - lg.max(0, keepdim=True).values).abs() + 4 * U
    bound = o * (a + (o * a).sum(0, keepdim=True) + (K + 1) * U)
    return o, bound, lg


def sum_and_range_ratio(o, K):
    """max |sum - 1| / ((K+1) 2^-23) over the pixels of o [K+1, ...] (K additions in the denominator and one rounding
    per quotient: (K+1) 2^-24 to first order, doubled for the higher-order terms); inf if a value leaves [0, 1]."""
    s = o.double().sum(0)
    if not bool(((o >= 0) & (o <= 1)).all()):
        return math.inf
    return float(((s - 1).abs() / ((K + 1) * 2.0 ** -23)).max()) if s.numel() else 0.0


def _sum_and_range(what, o, K):
    """Every pixel of [bg, objects] sums to 1 within (K+1) 2^-23, every value in [0, 1] (sum_and_range_ratio)."""
    ratio = sum_and_range_ratio(o, K)
    print(f"{what}: max |sum - 1| / bound = {ratio:.3g}")
    assert ratio <= 1.0, f"{what}: max |sum - 1| / bound = {ratio:.3g}"


def upsample4x_raw_reference(lg, H, W):
    """float64 sigmoid(bilinear x4(lg)) of logits lg [n, 1, h4, w4] and its bound: exact weights (multiples of 1/8),
    at most 4 roundings per corner term (|dv| <= 4u B|l|, B = bilinear of |l|), carried by sigma' = p (1 - p); then
    2 ulp of expf on exp(-v) scaled by 1 - p, and one rounding each for 1 + t and the reciprocal."""
    v = _bilinear(lg, H, W)
    p = torch.sigmoid(v)
    return p, p * (1 - p) * 4 * U * _bilinear(lg.abs(), H, W) + p * (2 * U + 4 * U * (1 - p))


# ------------------------------------------------------------------------------------------------ S2M resizes, pooling
def avgpool_reference(x):
    """fp64 mean over the pixels of x [n, c, h, w] and its bound for the kernel's summation order: each of 8 pixel
    groups sums its pixels sequentially, the 8 partials are added, the sum is multiplied by fl(1/hw)."""
    n, c, h, w = x.shape
    hw = h * w
    xd = x.double()
    mu = xd.mean((2, 3))
    s = xd.abs().sum((2, 3))
    return mu, (math.ceil(hw / 8) + 7) * U * s / hw + 2 * U * mu.abs()


def bilinear_reference(x, h, w):
    """fp64 F.interpolate(size=(h, w), align_corners=False) of x [n, c, hs, ws] and the kernels' bound on it: 5u of
    the weighted magnitude where the scale is a power of two (exact weights), 6u otherwise plus, per axis, the
    sample's offset from fl(in/out) and the source coordinate (3u (in + 1)) times the largest neighbour difference."""
    hs, ws = x.shape[-2:]
    xd = x.double()
    ref = F.interpolate(xd, size=(h, w), mode="bilinear", align_corners=False)
    mag = F.interpolate(xd.abs(), size=(h, w), mode="bilinear", align_corners=False)
    exact = all(math.log2(a / b).is_integer() for a, b in ((hs, h), (ws, w)))
    bound = (5 if exact else 6) * U * mag
    if not exact:
        dy = float(xd.diff(dim=2).abs().max()) if hs > 1 else 0.0
        dx = float(xd.diff(dim=3).abs().max()) if ws > 1 else 0.0
        bound = bound + 3 * U * (hs + 1) * dy + 3 * U * (ws + 1) * dx
    return ref, bound


def sigmoid_bound(p):
    """1 / (1 + expf(-x)) of an exact x: 2 ulp of expf scaled by 1 - sigma, one rounding each for the sum and the
    reciprocal (at most 6u relative)."""
    return p * (2 * U + 4 * U * (1 - p))


# ------------------------------------------------------------------------------------------------ stem gathers
def stem_images(frames, masks=None):
    """fp64 input images of a stem gather [N, cin, H, W] and the bound of each value.  frames alone: a batch of
    3- or 6-channel images.  frames [G, 3, H, W] with masks [G, K, H, W]: per object (group-major) the frame, its own
    mask and the exact sum of the other objects' masks.  The kernel adds the K - 1 other masks to 0 in object order,
    the first addition exact: |others - sum| <= (K - 2) u sum_{j != k} m_j.  Every other channel is one rounding of
    the fp32 operand to the map type, applied by the caller."""
    if masks is None:
        img = frames.double()
        return img, torch.zeros_like(img)
    G, K = masks.shape[:2]
    m = masks.double()
    imgs, bounds = [], []
    for k in range(K):
        others = torch.cat([m[:, :k], m[:, k + 1:]], 1).sum(1, keepdim=True)
        imgs.append(torch.cat([frames.double(), m[:, k:k + 1], others], 1))
        b = torch.zeros_like(imgs[-1])
        b[:, 4:] = max(K - 2, 0) * U * others
        bounds.append(b)
    N = G * K
    return torch.stack(imgs, 1).reshape(N, 5, *frames.shape[2:]), torch.stack(bounds, 1).reshape(N, 5, *frames.shape[2:])


def stem_matrix(img, kpad, s2d):
    """The gather of img [N, cin, H, W] as the kernels write it: HALO rows of the half-resolution output map, kpad
    columns.  49 taps: the F.unfold(7, stride 2, pad 3) windows in (ky, kx, c) order.  s2d (header formula):
    out[row(Y, X), py*8*cin + j*cin + c] = in[c, 2Y + py, 2X - 4 + j], zero outside the image.  Border rows and the
    pad columns are zero."""
    N, cin, H, W = img.shape
    ho, wo = H // 2, W // 2
    if s2d:
        p = F.pad(img, (4, 4))
        cols = torch.stack([p[:, :, py::2, j:j + 2 * wo:2] for py in range(2) for j in range(8)], 1)  # [N, 16, cin, ho, wo]
        cols = cols.permute(0, 3, 4, 1, 2).reshape(N, ho, wo, 16 * cin)
    else:
        cols = F.unfold(img, 7, padding=3, stride=2).reshape(N, cin, 49, ho, wo).permute(0, 3, 4, 2, 1)
        cols = cols.reshape(N, ho, wo, 49 * cin)
    out = torch.zeros((N, ho + 2, wo + 2, kpad), dtype=torch.float64, device=img.device)
    out[:, 1:-1, 1:-1, :cols.shape[-1]] = cols
    return out.reshape(-1, kpad)


def stem_reference(frame, masks, k0, n):
    """float64 space-to-depth memorize stem of objects [k0, k0 + n): channels (frame, own mask, sum of every OTHER
    mask of the K); out[row(Y,X), py*40 + j*5 + c] = in[c, 2Y+py, 2X-4+j]."""
    import abi_emulator
    f, m = frame.double().cpu(), masks.double().cpu()
    total = m.sum(0)
    inp = torch.cat([f.expand(n, -1, -1, -1), m[k0:k0 + n], total[None].expand(n, -1, -1, -1) - m[k0:k0 + n]], 1)
    H, W = f.shape[-2:]
    out = torch.zeros((n * (H // 2 + 2) * (W // 2 + 2), 80), dtype=torch.float64)
    abi_emulator._stem_s2d_frames(inp, out)
    return out


def stem_tolerance(ref, K, f16):
    """fp32 sequential sum of K - 1 masks in [0, 1]: (K - 1) u of the sum; fp16 storage adds one rounding (and half
    of its smallest subnormal step below 2^-14)."""
    return ref.abs() * ((K - 1) * U + (2.0 ** -11 if f16 else 0.0)) + (2.0 ** -24 if f16 else 0.0)
