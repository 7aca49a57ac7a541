"""TEST INFRASTRUCTURE: adversarial banks that drive the memory reads into their exact fallbacks, for
tests/test_gpu_memread_fallback.py and tests/test_memread_fallback_cpu.py.

A designed query reads one key channel: q = sqrt(128) * s * e_j with s a power of two, so q / sqrt(128) = s * e_j
exactly and its fp32 score of every slot is s * key[j] exactly (the fmaf chain adds zeros), in the kernels and in
numpy alike.  A quiet query is s * sqrt(128) * e_3 plus a small N(0, 0.1^2) part on the channels no construction
uses.  Channels 0-3 hold, in the first two tiles of every list, 64 values in [8, 12] per column half (the SUPPORT,
below every construction), so each list's own bound is high from the warm-up on and the lists of a quiet query, or of
a designed query on an object without its construction, stay short under every timing, while their top-k spreads
over all lists.  Query set g scales its designed queries by 2^g (SET_SCALE): every construction is invariant under a
power-of-two scale (the scores, margins, bucket maxima, bisection and histogram bins all scale exactly), but the
scores and the softmax read-out are not, so a read that serves a query with another set's query changes the result.  Each channel of a bank holds one construction, N(0, 1) elsewhere; quiet queries are N(0, 1) on the
channels no construction uses.  One slot per object holds ANCHOR * e_127, the longest key, so the TF32 margin of a
designed query is the same known value (2 * 1.05 * 2^-9 * ANCHOR, about 0.13) in every object.

Top-k read (k <= 64), in units of that margin M, `stream_slots(sp, h)` being the slots of split sp's column half h
(tests/memread_list_model.py restates the plan and the per-list bookkeeping):
  STREAM  channel 0: 640 bit-identical rows 20 * e_0 in tiles 1-5 of one (split 1, half 1) list (its first tile is
          N(0, 1), so that no query's own bound there sits at their score 0): the top of the order, more than
          LIST_LIMIT = 384 candidates in one list -> the tensor-core pass flags the query while streaming;
  SELECT  channel 1: 64 distinct near-ties (20 + i * 16 ulp, 0.48 M wide) in the first two tiles of every list:
          no list above 192, more than 1536 in band -> pass A flags the query;
  GLOBAL  channel 2: k distinct values 4 M above a shoulder of 48 slots at 20 in the first tile of every list; the top
          k sit in the first two lists and in too few buckets to raise the shared threshold above the shoulder:
          more than 1344 candidates above the staging cut, k after the bisection cut -> the global-memory filter, no
          flag.
Wide read (64 < k <= 1024), designed per channel for top_k (level-1 bins are octaves, level-2 bins 2^14 ulps):
  M0      k + 8 distinct values in [16, 32): mode 0;
  M10     2300 distinct values in [16, 32): mode 1, then 0;
  M12     2300 distinct values inside one level-2 bin at 16: mode 1, then 2 (the radix select over distinct scores);
  TIE2    k // 2 distinct values in [24, 32) and 2300 bit-identical rows at 20 straddling rank k: mode 1 then 2;
  TIE0    the same with 600 identical rows: mode 0 (the sort breaks the tie).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from memread_list_model import TS, TC_HALF, tc_plan, live_tps

H, W = 7, 9
HW = H * W
SQ = np.float32(math.sqrt(128))
ANCHOR = 32.0
LEVEL = 20.0
ULP20 = 2.0 ** -19                 # fp32 spacing in [16, 32)
CH_STREAM, CH_SELECT, CH_GLOBAL, CH_SUPPORT = 0, 1, 2, 3
QUIET0 = 8                         # the random part of quiet queries: channels 8 .. 126
QUIET_NOISE = 0.1
DESIGN_MARGIN = 2.0 * 1.05 * 2.0 ** -9 * ANCHOR * 1.0001

# query roles of the top-k reads: designed queries at both ends of the first 32-query exact tile, in the second tile,
# and in the partial last one; everything else quiet
TOPK_ROLES = {q: "stream" for q in (2, 9, 40)} | {q: "select" for q in (5, 20, 50, 62)} | {q: "global" for q in (11, 33)}
ROLE_CHANNEL = {"stream": CH_STREAM, "select": CH_SELECT, "global": CH_GLOBAL}


def stream_slots(sp, h, tps, live):
    """Slots of the list (split sp, column half h) in tile order, columns ascending."""
    t = np.arange(sp * tps, (sp + 1) * tps)[:, None] * TS + h * TC_HALF + np.arange(TC_HALF)[None, :]
    t = t.reshape(-1)
    return t[t < live]


def set_scale(g):
    """Scale of query set g's designed queries."""
    return float(2 ** g)


def topk_queries(sets, seed, roles=TOPK_ROLES):
    g = torch.Generator().manual_seed(seed)
    q = torch.zeros((sets, HW, 128))
    q[:, :, QUIET0:127] = QUIET_NOISE * torch.randn((sets, HW, 127 - QUIET0), generator=g)
    for st in range(sets):
        q[st, :, CH_SUPPORT] = float(SQ) * set_scale(st)
    for qi, r in roles.items():
        q[:, qi] = 0.0
        for st in range(sets):
            q[st, qi, ROLE_CHANNEL[r]] = float(SQ) * set_scale(st)
    return q


def _base(cap, live, seed, dups=True):
    """N(0, 1) keys and values; rows past `live` hold 8x the largest designed score in every channel (a stale row
    that took part would top every query); the first 2048 live rows come in bit-identical pairs; the anchor."""
    g = torch.Generator().manual_seed(seed)
    bk = torch.randn((cap, 128), generator=g)
    bv = torch.randn((cap, 512), generator=g)
    if dups:
        bk[1:2048:2] = bk[0:2047:2]
    bk[live:] = 8.0 * 32.0
    bk[live - 3] = 0.0
    bk[live - 3, 127] = ANCHOR
    return bk, bv


def topk_bank(cap, live, splits, tps, top_k, designs, seed):
    """One object's keys and values [cap, 128 / 512] with the top-k constructions in `designs`."""
    bk, bv = _base(cap, live, seed)
    ch = bk.numpy()
    nlists = [(sp, h) for sp in range(splits) for h in range(2) if stream_slots(sp, h, tps, live).size]
    rng = np.random.default_rng(seed)
    for sp, h in nlists:
        sl = stream_slots(sp, h, tps, live)
        sl = np.concatenate([sl[64:128], sl[TC_HALF + 64:TC_HALF + 128]])
        for c in (CH_STREAM, CH_SELECT, CH_GLOBAL, CH_SUPPORT):
            ch[sl, c] = (8.0 + 4.0 * rng.random(sl.size)).astype(np.float32)
    if "global" in designs:
        top = [s for sp, h in ((0, 0), (0, 1)) for s in stream_slots(sp, h, tps, live)[:2 * TC_HALF]
               if s % TC_HALF < -(-top_k // 4)]
        top = sorted(top, key=lambda s: (s % TC_HALF, s))[:top_k]
        assert len(top) == top_k
        for sp, h in nlists:
            ch[stream_slots(sp, h, tps, live)[64:112], CH_GLOBAL] = LEVEL
        for i, s in enumerate(sorted(top)):
            ch[s, CH_GLOBAL] = np.float32(LEVEL + 4 * DESIGN_MARGIN + 16 * i * ULP20)
    if "select" in designs:
        i = 0
        for sp, h in nlists:
            sl = stream_slots(sp, h, tps, live)
            for s in np.concatenate([sl[32:64], sl[TC_HALF + 32:TC_HALF + 64]]):
                ch[s, CH_SELECT] = np.float32(LEVEL + 16 * i * ULP20)
                i += 1
    if "stream" in designs:
        sl = stream_slots(1, 1, tps, live)[TC_HALF:6 * TC_HALF]
        assert sl.size == 5 * TC_HALF
        bk[torch.from_numpy(sl)] = 0.0
        bk[torch.from_numpy(sl), CH_STREAM] = LEVEL
    return bk, bv


# ------------------------------------------------------------------ layouts of the top-k launches
# (objects, live count of each object, query set of each object, constructions of each object)
def topk_layout(form, top_k, seed, sms=132):
    """Operands of one top-k fallback launch: dict(A=kwargs of the ops call, live, qset, designs, plan)."""
    if form == "groups":
        sizes, counts = [1, 2, 2], [24576, 23001, 23296]
        designs = [set(), set(), {"stream", "select", "global"}, {"stream"}, set()]
    elif form == "sets":
        sizes, counts = [2, 2], [24576, 23300]
        designs = [{"select"}, set(), {"stream", "select", "global"}, set()]
    else:  # scalar: q_div 2 (two query sets) or one set with a device-side count
        sizes = [2, 2] if form == "qdiv" else [3]
        counts = [24576] * len(sizes) if form == "qdiv" else [23800]
        designs = ([{"stream", "global"}, set(), set(), {"select"}] if form == "qdiv"
                   else [{"stream", "select", "global"}, set(), {"select"}])
    K = sum(sizes)
    cap = 24576
    splits, tps = tc_plan(cap, K, HW, sms)
    qset = [g for g, n in enumerate(sizes) for _ in range(n)]
    live = [counts[g] for g in qset]
    device = form != "qdiv"
    bks, bvs, tpss = [], [], []
    for o in range(K):
        t = live_tps(live[o], splits, tps, device)
        bk, bv = topk_bank(cap, live[o], splits, t, top_k, designs[o], seed + o)
        bks.append(bk)
        bvs.append(bv)
        tpss.append(t)
    qk = topk_queries(len(sizes), seed + 100)
    A = dict(bank_k=torch.stack(bks), bank_v=torch.stack(bvs), slots=cap, qk=qk, top_k=top_k)
    if form == "groups":
        A.update(counts=torch.tensor(counts, dtype=torch.int32),
                 first=torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32))
    elif form == "sets":
        A.update(counts=torch.tensor(counts, dtype=torch.int32))
    elif form == "qdiv":
        A.update(q_div=2)
    else:
        A.update(qk=qk[0], dyn_slots=torch.tensor(counts, dtype=torch.int32))
    return dict(A=A, live=live, qset=qset, designs=designs, splits=splits, tps=tpss)


def predicted_flags(layout):
    """Flagged queries each object's constructions call for: its stream and select queries."""
    n = 0
    for d in layout["designs"]:
        n += sum(1 for r in TOPK_ROLES.values() if r in d and r in ("stream", "select"))
    return n


def model_flags(layout):
    """[objects] dicts of memread_list_model.read_model over each object's live keys and its query set."""
    from memread_list_model import read_model
    A = layout["A"]
    qk = A["qk"] if A["qk"].dim() == 3 else A["qk"][None]
    out = []
    for o, (n, s) in enumerate(zip(layout["live"], layout["qset"])):
        keys = A["bank_k"][o, :n].numpy()
        qs = (qk[s].numpy().astype(np.float32) / SQ).astype(np.float32)
        out.append(read_model(keys, qs, A["top_k"], layout["splits"], layout["tps"][o]))
    return out


# ------------------------------------------------------------------ wide banks
WIDE_CHANNELS = ("M0", "M10", "M12", "TIE2", "TIE0")
WIDE_LEVEL2 = 16.0
WIDE_N = 2300                      # > WIDE_CAP: the band of a level-1 or level-2 bin


def wide_bank(cap, live, top_k, designed, seed):
    """One object's keys / values for the wide read; channel c of WIDE_CHANNELS holds its construction when
    `designed`, N(0, 1) otherwise.  Constructions use disjoint slots, placed at random."""
    bk, bv = _base(cap, live, seed, dups=False)
    if not designed:
        return bk, bv
    rng = np.random.default_rng(seed)
    perm = rng.permutation(live - 3)
    ch = bk.numpy()
    take = iter(np.split(perm, np.cumsum([top_k + 8, WIDE_N, WIDE_N, top_k // 2 + WIDE_N, top_k // 2 + 600])))

    def distinct(n, lo, width_ulps):
        return (np.float32(lo) + np.sort(rng.choice(width_ulps, n, replace=False)).astype(np.float64)
                * ULP20).astype(np.float32)

    sl = next(take)
    ch[sl, 0] = distinct(sl.size, 16.0, 2 ** 23)
    sl = next(take)
    ch[sl, 1] = distinct(sl.size, 16.0, 2 ** 23)
    sl = next(take)
    ch[sl, 2] = distinct(sl.size, WIDE_LEVEL2, 2 ** 14)
    for c in (3, 4):
        sl = next(take)
        ch[sl[:top_k // 2], c] = distinct(top_k // 2, 24.0, 2 ** 22)
        proto = bk[int(sl[top_k // 2])].clone()
        proto[c] = LEVEL
        bk[torch.from_numpy(np.sort(sl[top_k // 2:]))] = proto
    return bk, bv


# designed wide queries: channel c with scale s (a power of two: the same bins shifted, or the order reversed)
WIDE_ROLES = {q: (q % 5, (1.0, 2.0, -1.0, 0.5)[(q // 5) % 4]) for q in range(HW)}


def wide_queries(sets):
    q = torch.zeros((sets, HW, 128))
    for qi, (c, s) in WIDE_ROLES.items():
        for st in range(sets):
            q[st, qi, c] = float(SQ) * s * set_scale(st)
    return q


def wide_layout(form, top_k, seed):
    if form == "groups":
        sizes, counts = [1, 2, 2], [12288, 11001, 11776]
        designed = [False, False, True, True, False]
    else:
        sizes, counts = [2, 2], [12288, 11300]
        designed = [True, False, True, False]
    K = sum(sizes)
    cap = 12288
    qset = [g for g, n in enumerate(sizes) for _ in range(n)]
    live = [counts[g] for g in qset]
    parts = [wide_bank(cap, live[o], top_k, designed[o], seed + o) for o in range(K)]
    A = dict(bank_k=torch.stack([p[0] for p in parts]), bank_v=torch.stack([p[1] for p in parts]), slots=cap,
             qk=wide_queries(len(sizes)), top_k=top_k, counts=torch.tensor(counts, dtype=torch.int32))
    if form == "groups":
        A["first"] = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32)
    return dict(A=A, live=live, qset=qset, designed=designed)


def wide_predicted(layout):
    """[objects, HW] (mode, refined) from the exact fp32 scores of the designed queries."""
    from memread_list_model import wide_state
    A = layout["A"]
    return [[wide_state(s, A["top_k"]) for s in wide_scores(A["bank_k"][o, :n], layout["qset"][o]).values()]
            for o, n in enumerate(layout["live"])]


def wide_scores(keys, qset):
    """{query: exact fp32 scores over `keys` [live, 128]} of the designed wide queries of query set qset."""
    k = keys.cpu().numpy()
    return {q: (k[:, c] * np.float32(s * set_scale(qset))).astype(np.float32) for q, (c, s) in WIDE_ROLES.items()}


def topk_scores(keys, qset):
    """{query: exact fp32 scores over `keys` [live, 128]} of the designed top-k queries of query set qset."""
    k = keys.cpu().numpy()
    return {q: (k[:, ROLE_CHANNEL[r]] * np.float32(set_scale(qset))).astype(np.float32) for q, r in TOPK_ROLES.items()}


def expected_order(keys_col, top_k):
    """Indices of the exact top-k of one designed query: (score desc, slot asc), -1 past the live slots."""
    order = np.lexsort((np.arange(keys_col.size), -keys_col.astype(np.float64)))[:top_k]
    return np.concatenate([order, -np.ones(top_k - order.size, np.int64)])


def _prev_twin(keys):
    """[n] the previous slot whose key row is bit-identical, -1 if none."""
    _, inv = torch.unique(keys.cpu(), dim=0, return_inverse=True)
    prev = -np.ones(inv.numel(), np.int64)
    last = {}
    for s, g in enumerate(inv.tolist()):
        prev[s] = last.get(g, -1)
        last[g] = s
    return prev


def strict_check(A, live, qset, idx, val, designed):
    """What checked_read allows and these reads must not: equal scores listed out of slot order, a row selected
    without its bit-identical lower twin, and for each designed query (designed(o) -> {query: its fp32 scores over
    the live slots}) any other index list than the exact (score desc, slot asc) top-k, or other scores than its own."""
    idx, val = idx.cpu(), val.cpu()
    k = idx.shape[-1]
    v0, v1, i0, i1 = val[..., :-1], val[..., 1:], idx[..., :-1], idx[..., 1:]
    ok = (i1 < 0) | ((v0 >= v1) & ((v0 != v1) | (i0 < i1)))
    assert bool(ok.all()), "scores not descending, or equal scores not in ascending slot order"
    for o, n in enumerate(live):
        if qset[o] < 0:
            continue
        prev = _prev_twin(A["bank_k"][o, :n])
        sel = idx[o].numpy()
        for q in range(sel.shape[0]):
            s = sel[q][sel[q] >= 0]
            p = prev[s]
            assert np.isin(p[p >= 0], s).all(), f"object {o} query {q}: a row selected without its lower twin"
        for q, col in designed(o).items():
            want = expected_order(col, k)
            assert np.array_equal(sel[q], want), (f"object {o} query {q}: {sel[q][:8]}... is not the exact top-{k} "
                                                 f"{want[:8]}...")
            got = val[o, q].numpy()[want >= 0]
            assert np.array_equal(got, col[want[want >= 0]]), f"object {o} query {q}: scores not its exact fp32 scores"
