"""CPU model of the candidate lists of the memory read's tensor-core pass (mivos_b200/csrc/memread_tc.cu) — test
infrastructure, like the oracle it imports.  It replays the kernel's bookkeeping in numpy on real key / query
features of the oracle network: streams = (split of the slot axis) x (column half of a 256-slot tile); per stream
NB bucket maxima (bucket = column mod NB), thresholds refreshed after the warm-up tiles, every 4th tile and at the
end, shared across streams through a max (`tau_g`), optionally tightened by the PAIR rule (min over the two halves
of their ceil(k/2)-th bucket maximum); emission of every score >= threshold - margin from the tiles after the
warm-up, compaction when a list passes 384, replay of the warm-up tiles at the end.

  python tests/memread_list_model.py K frames top_k [pair]     e.g.  3 26 50 1   (cfg-3 at its mean bank)

Numbers this produced on the synthetic cfg-3 clip (seeded random weights; margin 0.23 for a score spread of 0.77):
  k-th-of-64 thresholds only : 1440-1730 candidates per query in the lists, 930 of them within the final threshold,
                               5 % of the queries above the old per-list cap of 224 -> 3/4 of the exact fallback's tiles
  + PAIR rule                : 380 within the final threshold (the in-band minimum is 117), none flagged
(the fallback decision moved into the selection stage)."""
import math
import sys

import numpy as np


def features(K, frames, seed=1234):
    import torch
    sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
    from mivos_b200 import synth
    from oracle import stm_oracle as O
    torch.set_grad_enabled(False)
    psd = synth.make_prop_state_dict()
    images, mask = synth.synthetic_clip(frames + 1, 480, 854, K, seed=seed)
    imgs, _ = O.pad_divide_by(images, 16, images.shape[-2:])
    m, _ = O.pad_divide_by(mask, 16, mask.shape[-2:])
    keys = [O.memorize(psd, imgs[:, t], m[1:])[0] for t in range(frames)]
    qk = O.get_query_values(psd, imgs[:, frames])[3]
    return torch.cat(keys, 2).numpy(), qk.numpy()


def pair_bound(m_a, m_b, k):
    """min over the two halves of their ceil(k/2)-th largest bucket maximum: the halves saw disjoint slots, so
    together they hold k scores >= it — a lower bound of the k-th largest score of their union."""
    kh = (k + 1) // 2
    a = -np.sort(-m_a, axis=-1)[..., kh - 1]
    b = -np.sort(-m_b, axis=-1)[..., kh - 1]
    return np.minimum(a, b)


def run(mk, qk, top_k, pair, verbose=True):
    Kk, CK, T, h, w = mk.shape
    hw, slots = h * w, T * h * w
    keys = mk.reshape(Kk, CK, slots).transpose(0, 2, 1)
    q = (qk.reshape(CK, hw).T / np.float32(math.sqrt(128))).astype(np.float32)
    NB, TS, CAP = (32 if top_k <= 32 else 64), 256, 512
    qtiles, tiles = (hw + 127) // 128, (slots + TS - 1) // TS
    s = max(1, min(132 // (qtiles * Kk), max(1, tiles // 4), 16))  # one wave on the 132 SMs of an H100
    tps = (tiles + s - 1) // s
    splits = (tiles + tps - 1) // tps
    out = []
    for obj in range(Kk):
        S = q @ keys[obj].T
        margin = 2.0 * 1.05 * 0.001953125 * np.linalg.norm(q, axis=1) * 1.0001 * math.sqrt((keys[obj] ** 2).sum(1).max() * 1.0001)
        kth_true = -np.sort(-S, axis=1)[:, top_k - 1]
        ns = splits * 2
        m = np.full((ns, hw, NB), -np.inf, np.float32)
        tau_g = np.full(hw, -3e38, np.float32)
        tau_emit = np.full((ns, hw), -np.inf, np.float32)
        cnt = np.zeros((ns, hw), np.int64)
        for i in range(tps):
            for sp in range(splits):
                nloc = min(tiles, (sp + 1) * tps) - sp * tps
                if i >= nloc:
                    continue
                warm = min(2, nloc)
                for half in range(2):
                    st = sp * 2 + half
                    c0 = (sp * tps + i) * TS + half * 128
                    cols = S[:, c0:min(c0 + 128, slots)]
                    for cc in range(0, cols.shape[1], 32):
                        off = 32 if (NB == 64 and ((cc // 32) & 1)) else 0
                        blk = cols[:, cc:cc + 32]
                        m[st][:, off:off + blk.shape[1]] = np.maximum(m[st][:, off:off + blk.shape[1]], blk)
                    if i >= warm:
                        cnt[st] += (cols >= tau_emit[st][:, None]).sum(1)
            for sp in range(splits):
                nloc = min(tiles, (sp + 1) * tps) - sp * tps
                if i >= nloc:
                    continue
                warm = min(2, nloc)
                if (i + 1 == warm) or (i + 1 > warm and ((i + 1 - warm) & 3) == 0) or (i + 1 == nloc):
                    if pair:
                        tau_g = np.maximum(tau_g, np.maximum(pair_bound(m[sp * 2], m[sp * 2 + 1], top_k), -3e38))
                    for half in range(2):
                        st = sp * 2 + half
                        tau_g = np.maximum(tau_g, np.maximum(-np.sort(-m[st], axis=1)[:, min(top_k, NB) - 1], -3e38))
                        tau_emit[st] = np.maximum(tau_g - margin, -3e38)
        assert (tau_g <= kth_true + 1e-6).all(), "a threshold above the true k-th largest score"
        inband = (S >= (tau_g - margin)[:, None]).sum(1)
        ideal = (S >= (kth_true - margin)[:, None]).sum(1)
        out.append((cnt.sum(0).mean(), inband.mean(), inband.max(), ideal.mean()))
        if verbose:
            print(f"object {obj}: {ns} lists/query, emitted {cnt.sum(0).mean():.0f} per query (before compaction / replay), "
                  f"within the final threshold {inband.mean():.0f} (max {inband.max()}), in-band minimum {ideal.mean():.0f}")
    return out



# ------------------------------------------------------------------ the read on arbitrary scores
# The same bookkeeping on any approximate score matrix, with the list capacity, compaction and the selection stage
# (pass A) of the kernels, for the fallback tests (tests/test_memread_fallback_cpu.py, tests/test_gpu_memread_fallback.py).
# Which bound another CTA has published when is a matter of timing, so the model gives bounds that hold for every
# timing:
#   * tau_g, the shared threshold the selection stage reads, is the maximum over all streams of their FINAL own and
#     pair bounds (bucket maxima only grow): it does not depend on timing;
#   * every slot with approx >= tau_g - margin is emitted into its list and never compacted away, so a list ends at
#     least that long (`low`); one that long above LIST_LIMIT flags its query;
#   * without sharing a stream's threshold is lowest, so its lists are longest: `high` is the largest count, over
#     every overflow check, of the emitted entries a compaction would keep.  At most LIST_LIMIT: no flag.
#     `high_tf32` is the same count with the threshold one more margin lower: the scores and the bounds of the GPU may
#     differ from the model's TF32 operands by their rounding, at most half a margin each, so at most LIST_LIMIT there
#     means no flag whatever the rounding.
TS, TC_HALF, LIST_CAP = 256, 128, 512
LIST_LIMIT = LIST_CAP - TC_HALF        # a list longer than this after compaction flags its query
SEL_CAP, STAGE_LIMIT = 1024, 896       # survivors pass A re-scores; staging stops above STAGE_LIMIT
MARGIN_FACTOR = np.float32(2.0 * 1.05 * 0.001953125)
LOWEST = np.float32(-3.0e38)


def tf32(x):
    """fp32 -> TF32 operand (the tensor cores read the top 19 bits)."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)
    return b.view(np.float32)


def tc_plan(slots, k_objects, hw, sms):
    """(splits, tiles_per_split) of the tensor-core plan (memread_plan)."""
    qtiles, tiles = -(-hw // 128), -(-slots // TS)
    s = min(sms // (qtiles * k_objects), max(tiles // 4, 1))
    s = min(max(s, 1), 16)
    tps = -(-tiles // s)
    return -(-tiles // tps), tps


def live_tps(live, splits, tps, device_count):
    """Tiles per split of a read over `live` slots: a device-side count derives them from the launch's splits."""
    return -(-(-(-live // TS)) // splits) if device_count else tps


def margin(keys, qs):
    """Per-query TF32 margin of one object (keys [n,128] live rows, qs [nq,128] scaled queries), as the kernels
    round it."""
    qn = np.sqrt((qs.astype(np.float32) ** 2).sum(1, dtype=np.float32)) * np.float32(1.0001)
    km = (keys.astype(np.float32) ** 2).sum(1, dtype=np.float32).max() * np.float32(1.0001)
    return (MARGIN_FACTOR * qn.astype(np.float32) * np.sqrt(np.float32(km))).astype(np.float32)


def approx_scores(keys, qs):
    """[nq, n] scores of TF32 operands, accumulated in float64, rounded to fp32."""
    return (tf32(qs).astype(np.float64) @ tf32(keys).astype(np.float64).T).astype(np.float32)


def _kth(m, k):
    return -np.sort(-m, axis=-1)[..., k - 1]


def lists_model(S, mg, top_k, splits, tps):
    """S [nq, n] approximate scores of one object, mg [nq] margins.  Returns tau_g [nq] and, per list
    (split * 2 + half), `low`, `high` and `high_tf32` [nq, 2 * splits] as described above."""
    nq, n = S.shape
    tiles = -(-n // TS)
    NB, kh = (32 if top_k <= 32 else 64), (top_k + 1) // 2
    pad = np.full((nq, splits * tps * TS), -np.inf, np.float32)
    pad[:, :n] = S
    low = np.zeros((nq, 2 * splits), np.int64)
    high = np.zeros((nq, 2 * splits), np.int64)
    high_tf32 = np.zeros((nq, 2 * splits), np.int64)
    tau_g = np.full(nq, LOWEST, np.float32)
    views = []
    for sp in range(splits):
        nloc = min(tiles, (sp + 1) * tps) - sp * tps
        if nloc <= 0:
            views.append(None)
            continue
        V = pad[:, sp * tps * TS:(sp * tps + nloc) * TS].reshape(nq, nloc, 2, TC_HALF)
        views.append(V)
        fin = [V[:, :, h].reshape(nq, nloc * TC_HALF // NB, NB).max(1) for h in range(2)]
        pair = np.minimum(_kth(fin[0], kh), _kth(fin[1], kh))
        tau_g = np.maximum(tau_g, np.maximum(np.maximum(_kth(fin[0], top_k), _kth(fin[1], top_k)), pair))
        # no sharing: the longest lists
        warm = min(2, nloc)
        m = [np.full((nq, NB), -np.inf, np.float32) for _ in range(2)]
        emit = [np.full(nq, -np.inf, np.float32) for _ in range(2)]
        done = []
        for i in range(nloc + warm):
            li = i if i < nloc else i - nloc
            if i < nloc:
                for h in range(2):
                    m[h] = np.maximum(m[h], V[:, li, h].reshape(nq, TC_HALF // NB, NB).max(1))
            if i >= warm:
                done.append(li)
            if (i + 1 == warm) or (i + 1 > warm and ((i + 1 - warm) & 3) == 0) or (i + 1 == nloc):
                p = np.minimum(_kth(m[0], kh), _kth(m[1], kh))
                for h in range(2):
                    t = np.maximum(_kth(m[h], top_k), p)
                    emit[h] = np.maximum(t - mg, LOWEST)
            if done:
                for h in range(2):
                    c = (V[:, done, h] >= emit[h][:, None, None]).sum((1, 2))
                    high[:, 2 * sp + h] = np.maximum(high[:, 2 * sp + h], c)
                    c = (V[:, done, h] >= (emit[h] - mg)[:, None, None]).sum((1, 2))
                    high_tf32[:, 2 * sp + h] = np.maximum(high_tf32[:, 2 * sp + h], c)
    for sp, V in enumerate(views):
        if V is not None:
            for h in range(2):
                low[:, 2 * sp + h] = (V[:, :, h] >= (tau_g - mg)[:, None, None]).sum((1, 2))
    return tau_g, low, high, high_tf32


def select_model(S, mg, top_k, tau_g, low, tps):
    """Pass A of one object's queries on the lists that hold every slot >= tau_g - margin (`low` of them per list):
    `staged` (candidates at or above the staging cut; above STAGE_LIMIT the rest is filtered from global memory),
    `band` (a lower bound of the survivors: approx >= k-th approx - margin), `survivors` after the kernel's bisection,
    replayed in fp32 on the full staged set, and `survivors_max`, an upper bound for any staging order.  Staging reads
    the lists in order and goes on while it holds at most STAGE_LIMIT, so every list up to the last one whose running
    count stays at or below STAGE_LIMIT is staged whole; the bisection stops at a value with at most 2k + 8 staged
    candidates above it, so at or above the (2k + 9)-th largest of that prefix."""
    nq, n = S.shape
    half = np.float32(0.5)
    cut0 = (tau_g - mg).astype(np.float32)
    staged = (S >= cut0[:, None]).sum(1)
    band = (S >= (_kth(S, top_k) - mg)[:, None]).sum(1)
    slot = np.arange(n)
    list_of = 2 * (slot // TS // tps) + (slot % TS) // TC_HALF
    surv = np.zeros(nq, np.int64)
    surv_max = np.zeros(nq, np.int64)
    for q in range(nq):
        v = S[q][S[q] >= cut0[q]]
        nn = v.size
        kk0 = min(top_k, nn)
        lo, hi = (v.min(), v.max()) if nn else (np.float32(np.inf), np.float32(-np.inf))
        limit = 2 * kk0 + 8
        for _ in range(26):
            if nn <= limit:
                break
            mid = np.float32(half * lo + half * hi)
            if not (mid > lo) or not (mid < hi):
                break
            c = int((v >= mid).sum())
            if c >= kk0:
                lo = mid
                if c <= limit:
                    break
            else:
                hi = mid
        cut = max(np.float32(lo - mg[q]), cut0[q])
        surv[q] = int((S[q] >= cut).sum())
        whole = int((np.cumsum(low[q]) <= STAGE_LIMIT).sum())
        pre = np.sort(S[q][(list_of < whole) & (S[q] >= cut0[q])])[::-1]
        bound = cut0[q] if nn <= limit or pre.size <= limit else max(np.float32(pre[limit] - mg[q]), cut0[q])
        surv_max[q] = int((S[q] >= bound).sum())
    return staged, band, surv, surv_max


def read_model(keys, qs, top_k, splits, tps):
    """Everything the fallback tests predict for one object: dict of [nq] arrays and the per-list bounds."""
    mg = margin(keys, qs)
    S = approx_scores(keys, qs)
    tau_g, low, high, high_tf32 = lists_model(S, mg, top_k, splits, tps)
    staged, band, surv, surv_max = select_model(S, mg, top_k, tau_g, low, tps)
    stream = low.max(1) > LIST_LIMIT
    return dict(margin=mg, tau_g=tau_g, low=low, high=high, high_tf32=high_tf32, staged=staged, band=band, survivors=surv,
                survivors_max=surv_max,
                stream_flag=stream, select_flag=~stream & (surv > SEL_CAP), flag=stream | (surv > SEL_CAP),
                global_path=~stream & (staged > STAGE_LIMIT))


# ------------------------------------------------------------------ the wide read's thresholds
WIDE_CAP, WIDE_BINS = 2048, 512


def score_key(s):
    """float_ordered(s) ^ 0x80000000 as uint32 (memread_wide.cu)."""
    b = np.ascontiguousarray(s, dtype=np.float32).view(np.int32)
    fo = np.where(b >= 0, b, b ^ np.int32(0x7FFFFFFF))
    return (fo ^ np.int32(-2 ** 31)).view(np.uint32)


def _digit(hist, need):
    """(digit, slots above it, slots in it) of the bin holding rank `need` from the top, None if fewer slots."""
    above = np.concatenate([np.cumsum(hist[::-1])[::-1][1:], [0]])
    for d in range(len(hist) - 1, -1, -1):
        if above[d] < need <= above[d] + hist[d]:
            return d, int(above[d]), int(hist[d])
    return None


def wide_state(scores, top_k):
    """(mode, refined) of one query of the wide read from its exact fp32 scores over the live slots: mode 0 (emit) or 2
    (exact fallback); refined: the level-2 sweep ran (mode 1 on the way)."""
    u = score_key(scores)
    h1 = np.bincount(u >> 23, minlength=WIDE_BINS)
    r = _digit(h1, top_k)
    if r is None:
        return (0 if u.size <= WIDE_CAP else 2), False
    d1, above, cnt = r
    if above + cnt <= WIDE_CAP:
        return 0, False
    h2 = np.bincount((u[(u >> 23) == d1] >> 14) & (WIDE_BINS - 1), minlength=WIDE_BINS)
    d2, above2, cnt2 = _digit(h2, top_k - above)
    return (0 if above + above2 + cnt2 <= WIDE_CAP else 2), True


if __name__ == "__main__":
    K, frames, top_k = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    mk, qk = features(K, frames)
    run(mk, qk, top_k, bool(int(sys.argv[4])) if len(sys.argv) > 4 else True)
