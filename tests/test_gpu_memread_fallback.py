"""GPU: the memory reads' exact fallbacks in every production form, checked against float64.

The constructions of tests/memread_fallback_cases.py drive the top-k read (k <= 64) into its three rescue paths —
the tensor-core pass flagging a query whose list overflows while streaming, selection pass A flagging a query with
more than 1024 candidates in band, and the global-memory filter of candidates past the staging capacity — and the wide
read (64 < k <= 1024) into its level-2 refinement (mode 1) and its radix select (mode 2), with flagged and unflagged
objects, queries and groups in one launch.  Every read goes through `memory_census.checked_read` (float64 index sets
outside TIE_EPS, the read-out over the kernel's own set, bit equality with the want_topk and MEMREAD_EXACT_SIMT
re-runs, finite windows, untouched bytes outside the window), and on top of it:
  * every designed query, whose fp32 scores are exactly one key channel, selects exactly the (score desc, slot asc)
    top-k, ties to the lowest slots; every query lists equal scores in ascending slot order and never selects a row
    whose bit-identical lower twin it left out;
  * each case proves its branch ran: mivos_memory_read_stats reports exactly the flagged queries the construction
    (and the CPU model of tests/memread_list_model.py) predicts; the candidate lists of every GLOBAL query, read from
    the workspace, hold more entries than staging takes (the global-memory filter's precondition); and the wide read's
    per-query state in the workspace holds the predicted mode;
  * for k <= 64 the wide read gives the top-k read's bits on the same banks.
Each case prints one row: form, k, counts, predicted and observed flags (or wide modes), worst err/bound."""
import ctypes
from collections import Counter

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import memory_census as MC  # noqa: E402
import memread_fallback_cases as C  # noqa: E402
import memread_list_model as LM  # noqa: E402
from mivos_b200 import _lib, ops  # noqa: E402

TOPK_FN = {"qdiv": ("memory_read", ops.memory_read), "scalar": ("memory_read", ops.memory_read),
           "sets": ("memory_read_sets", ops.memory_read_sets), "groups": ("memory_read_groups", ops.memory_read_groups)}
WIDE_FN = {"qdiv": ops.memory_read_wide, "scalar": ops.memory_read_wide, "sets": ops.memory_read_wide_sets,
           "groups": ops.memory_read_wide_groups}
WIDE_CENSUS = {"sets": ("memory_read_wide_sets", ops.memory_read_wide_sets),
               "groups": ("memory_read_wide_groups", ops.memory_read_wide_groups)}


def _dev(A, dev):
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in A.items()}


def _out(K, kind, dev):
    """pm32: pixel-major fp32 [K, HW, 640], window at channel 64; halo32 / halo16: a `cat` map of K maps at channel
    256, the leading view of an allocation one map larger; every byte a sentinel."""
    if kind == "pm32":
        return dict(out=torch.full((K, C.HW, 640), -3.5, device=dev), out_coff=64)
    dt = torch.float16 if kind == "halo16" else torch.float32
    parent = torch.full((K + 1, C.H + 2, C.W + 2, 1024), -3.5, dtype=dt, device=dev)
    return dict(out=parent[:K], out_coff=256, halo_hw=(C.H, C.W))


def _stats(ws, K, slots, k):
    st = (ctypes.c_int64 * 4)()
    _lib.check(_lib.lib().mivos_memory_read_stats(ctypes.c_void_p(ws.data_ptr()), K, slots, C.HW, k, st),
               "mivos_memory_read_stats")
    return list(st)


def _list_totals(ws, K, splits):
    """[K, HW] candidate-list entries of each query of the last top-k read in `ws`: the tensor-core plan's lengths
    follow its lists (kTcCandCap = 512 entries of 8 bytes per list, 4 KB of alignment slack), 2 * splits per query."""
    nlists = 2 * splits
    off_cnt = K * C.HW * nlists * 512 * 8 + 4096
    cnt = ws[off_cnt:off_cnt + K * C.HW * nlists * 4].cpu().view(torch.int32).reshape(K, C.HW, nlists)
    return cnt.sum(-1).numpy()


def _sync():
    torch.cuda.synchronize()
    _lib.poll_kernel_error()


TOPK_CASES = [("qdiv", 20, "pm32"), ("qdiv", 64, "halo16"), ("scalar", 50, "halo16"), ("scalar", 64, "pm32"),
              ("sets", 20, "halo32"), ("sets", 64, "halo16"), ("groups", 20, "halo16"), ("groups", 50, "pm32"),
              ("groups", 64, "halo32")]


@pytest.mark.parametrize("form,k,out", TOPK_CASES, ids=[f"{f}-k{k}-{o}" for f, k, o in TOPK_CASES])
def test_topk_fallback_paths(dev, form, k, out):
    L = C.topk_layout(form, k, seed=7)
    K = len(L["live"])
    predicted = C.predicted_flags(L)
    model = C.model_flags(L)
    assert sum(int(m["flag"].sum()) for m in model) == predicted
    A = _dev(L["A"], dev)
    ws = torch.zeros(ops.memory_read_workspace_bytes(K, A["slots"], C.HW, k), dtype=torch.uint8, device=dev)
    A.update(_out(K, out, dev), workspace=ws)
    name, fn = TOPK_FN[form]
    rec = MC.checked_read(name, fn, A)
    _sync()
    st = rec["stats"]
    assert st[3] == L["splits"], st
    assert 0 < predicted < K * C.HW
    assert st[2] == predicted, f"{st[2]} queries on the exact fallback, {predicted} predicted"
    # the global-memory filter: every GLOBAL query's lists hold more candidates than staging takes, at least the
    # model's count above the staging cut (the production read's list lengths, in its workspace)
    # (list lengths depend on when each CTA sees the shared threshold, so they are checked against the statistics
    # of the same read's workspace)
    st_ws = _stats(ws, K, A["slots"], k)
    assert st_ws[2] == predicted, st_ws
    total = _list_totals(ws, K, L["splits"])
    flagged = np.stack([m["flag"] for m in model])
    assert int(total[~flagged].sum()) == st_ws[0] and int(total[~flagged].max()) == st_ws[1], (st_ws, "list lengths")
    glob = [(o, q) for o in range(K) if "global" in L["designs"][o] for q, r in C.TOPK_ROLES.items() if r == "global"]
    for o, q in glob:
        assert total[o, q] > LM.STAGE_LIMIT and total[o, q] >= model[o]["staged"][q], (o, q, int(total[o, q]))
    # the selected sets and scores, and the wide read's bits on the same banks
    o1, i1, v1 = fn(**dict(A, out=A["out"].clone(), want_topk=True))
    o2, i2, v2 = WIDE_FN[form](**dict(A, out=A["out"].clone(), want_topk=True))
    _sync()
    assert torch.equal(i1, i2) and torch.equal(v1, v2) and torch.equal(o1, o2), "the wide read differs"
    C.strict_check(A, L["live"], L["qset"], i1, v1,
                   lambda o: C.topk_scores(A["bank_k"][o, :L["live"][o]], L["qset"][o]))
    paths = Counter()
    for m in model:
        paths.update(stream=int(m["stream_flag"].sum()), select=int(m["select_flag"].sum()),
                     global_filter=int(m["global_path"].sum()))
    print(f"\ntop-k {form:6s} k {k:2d} {out:6s} counts {rec['counts']} first {rec['first']}: flagged predicted "
          f"{predicted} observed {st[2]} of {K * C.HW} (model: {paths['stream']} streaming, {paths['select']} pass A; "
          f"{paths['global_filter']} through the global filter), GLOBAL list entries "
          f"{sorted(int(total[o, q]) for o, q in glob)} > {LM.STAGE_LIMIT}, err/bound {rec['ratio']:.3g}")


def _wide_offsets(K, hw):
    """wide_plan's workspace offsets: histograms | counts | WideState {cut, d1, above, mode} | candidate regions."""
    nq = K * hw
    off_cnt = nq * 512 * 4
    off_state = off_cnt + ((nq * 4 + 255) & ~255)
    off_cand = off_state + ((nq * 16 + 255) & ~255)
    return off_state, off_cand + nq * 2048 * 8


WIDE_CASES = [("sets", 65, "pm32"), ("sets", 256, "halo16"), ("sets", 1024, "halo32"), ("groups", 65, "halo16"),
              ("groups", 256, "halo32"), ("groups", 1024, "pm32")]


@pytest.mark.parametrize("form,k,out", WIDE_CASES, ids=[f"{f}-k{k}-{o}" for f, k, o in WIDE_CASES])
def test_wide_refinement_and_radix_select(dev, form, k, out):
    L = C.wide_layout(form, k, seed=3)
    K = len(L["live"])
    pred = C.wide_predicted(L)
    off_state, nbytes = _wide_offsets(K, C.HW)
    assert ops.memory_read_wide_workspace_bytes(K, L["A"]["slots"], C.HW, k) == nbytes
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    A = _dev(L["A"], dev)
    A.update(_out(K, out, dev), workspace=ws)
    name, fn = WIDE_CENSUS[form]
    rec = MC.checked_read(name, fn, A)
    _sync()
    state = ws[off_state:off_state + K * C.HW * 16].cpu().view(torch.int32).reshape(K, C.HW, 4)
    got = [[(int(state[o, q, 3]), int(state[o, q, 1]) != 0) for q in range(C.HW)] for o in range(K)]
    assert got == pred, [(o, q, got[o][q], pred[o][q]) for o in range(K) for q in range(C.HW) if got[o][q] != pred[o][q]][:8]
    kinds = Counter(m for row in got for m in row)
    assert {(0, False), (0, True), (2, True)} <= set(kinds), kinds
    _, i1, v1 = fn(**dict(A, out=A["out"].clone(), workspace=None, want_topk=True))
    _sync()
    C.strict_check(A, L["live"], L["qset"], i1, v1,
                   lambda o: C.wide_scores(A["bank_k"][o, :L["live"][o]], L["qset"][o]))
    print(f"\nwide {form:6s} k {k:4d} {out:6s} counts {rec['counts']} first {rec['first']}: modes predicted = observed: "
          f"{kinds[(0, False)]} mode 0, {kinds[(0, True)]} mode 1 -> 0, {kinds[(2, True)]} mode 1 -> 2, "
          f"{kinds[(2, False)]} mode 0 -> 2; err/bound {rec['ratio']:.3g}")


# ------------------------------------------------------------------ device counts below k
@pytest.mark.parametrize("k", [20, 64, 100])
def test_device_count_below_k_selects_every_live_slot(dev, k):
    """Per-set and grouped launches sized for k accept live counts below k (and 0): both reads select every live
    slot, pad topk_idx with -1 and topk_val with 0, and read out the softmax over the live slots (zeros for none);
    for k <= 64 the top-k read (both candidate generators) and the wide read give the same bits, in both forms."""
    g = torch.Generator().manual_seed(k)
    cap = 4 * C.HW + 300
    K = 4
    bk = torch.randn((K, cap, 128), generator=g).to(dev)
    bv = torch.randn((K, cap, 512), generator=g).to(dev)
    qk = torch.randn((K, C.HW, 128), generator=g).to(dev)
    # grouped: groups [0, 1), [1, 3), [3, 4) with counts k - 1, 1, 0; per set: one object per set, counts k - 1, 1, 0, 3
    layouts = {
        "groups": (lambda fn, **kw: fn(bk, bv, cap, qk[:3], k, torch.full((K, C.HW, 512), 9.0, device=dev),
                                       torch.tensor([k - 1, 1, 0], dtype=torch.int32, device=dev),
                                       torch.tensor([0, 1, 3, 4], dtype=torch.int32, device=dev), want_topk=True, **kw),
                   (ops.memory_read_groups, ops.memory_read_wide_groups), [k - 1, 1, 1, 0], [0, 1, 1, 2]),
        "sets": (lambda fn, **kw: fn(bk, bv, cap, qk, k, torch.full((K, C.HW, 512), 9.0, device=dev),
                                     torch.tensor([k - 1, 1, 0, 3], dtype=torch.int32, device=dev), want_topk=True,
                                     **kw),
                 (ops.memory_read_sets, ops.memory_read_wide_sets), [k - 1, 1, 0, 3], [0, 1, 2, 3]),
    }
    for form, (call, (topk_fn, wide_fn), live, qset) in layouts.items():
        reads = [call(wide_fn)]
        if k <= 64:
            reads += [call(topk_fn), call(topk_fn, algo=ops.MEMREAD_EXACT_SIMT)]
        _sync()
        for r in reads[1:]:
            assert all(torch.equal(a, b) for a, b in zip(reads[0], r)), f"{form}: the reads disagree"
        out, idx, val = reads[0]
        for o in range(K):
            n = live[o]
            assert bool((idx[o, :, n:] == -1).all()) and bool((val[o, :, n:] == 0).all()), (form, o)
            if n == 0:
                assert bool((out[o] == 0).all()), (form, o)
                continue
            assert torch.equal(idx[o, :, :n].sort(1)[0].long().cpu(), torch.arange(n).expand(C.HW, n)), (form, o)
            q = MC.scaled_q(qk[qset[o]])
            S = q @ bk[o, :n].double().t()
            ref = torch.softmax(S, 1) @ bv[o, :n].double()
            assert float((out[o].double() - ref).abs().max()) <= MC.RANGE_TERM * float(ref.abs().max()), (form, o)
        print(f"\n{form} counts {live} below k = {k}: every live slot selected, -1 / 0 padding, zeros for a count of 0"
              + (", top-k (both generators) and wide reads bit-equal" if k <= 64 else ""))


# ------------------------------------------------------------------ graph replay
def test_graph_replay_clears_stale_flags(dev):
    """One captured scalar read replayed while the device count grows: no flagged query (the near-tie cluster is not
    live), the SELECT construction's flags, none again (a block of larger keys past the cluster), and back.  Each
    replay gives the bits of the eager read at that count, so the captured memset clears the flags of the last one."""
    from memread_list_model import read_model, tc_plan, live_tps
    k, K, cap = 20, 2, 24576
    n_mid = 23001
    splits, tps = tc_plan(cap, K, C.HW, 132)
    t_mid = live_tps(n_mid, splits, tps, True)
    bks, bvs = [], []
    for o in range(K):
        bk, bv = C.topk_bank(cap, n_mid, splits, t_mid, k, {"select"}, seed=50 + o)
        bk[n_mid:] = torch.randn((cap - n_mid, 128), generator=torch.Generator().manual_seed(60 + o))
        bk[n_mid:n_mid + 256, C.CH_SELECT] = torch.from_numpy(
            (np.float32(C.LEVEL + 8 * C.DESIGN_MARGIN) + np.arange(256, dtype=np.float32) * np.float32(16 * C.ULP20)))
        bks.append(bk)
        bvs.append(bv)
    bk, bv = torch.stack(bks), torch.stack(bvs)
    qk = C.topk_queries(1, 70)[0]
    counts = (30, n_mid, cap)
    pred = {}
    for n in counts:
        qs = (qk.numpy() / C.SQ).astype(np.float32)
        pred[n] = sum(int(read_model(bk[o, :n].numpy(), qs, k, splits, live_tps(n, splits, tps, True))["flag"].sum())
                      for o in range(K))
    assert pred[counts[0]] == 0 and pred[counts[1]] > 0 and pred[counts[2]] == 0, pred
    bk, bv, qk = bk.to(dev), bv.to(dev), qk.to(dev)
    dyn = torch.zeros(1, dtype=torch.int32, device=dev)
    nbytes = ops.memory_read_workspace_bytes(K, cap, C.HW, k)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    out = torch.zeros((K, C.HW, 512), device=dev)
    idx = torch.zeros((K, C.HW, k), dtype=torch.int32, device=dev)
    val = torch.zeros((K, C.HW, k), device=dev)

    def call():
        _lib.check(_lib.lib().mivos_memory_read(ops._ptr(bk), ops._ptr(bv), cap, K, cap, ops._ptr(qk), C.HW, 0, k,
                                                ops._ptr(out), 512, 0, 0, 0, ops._ptr(idx), ops._ptr(val),
                                                ops._ptr(ws), nbytes, ops.MEMREAD_AUTO, ops._ptr(dyn), 0,
                                                ops._stream()), "mivos_memory_read")

    want = {}
    for n in counts:
        ops.store_i32(dyn, n)
        call()
        _sync()
        assert _stats(ws, K, cap, k)[2] == pred[n], (n, _stats(ws, K, cap, k), pred[n])
        want[n] = (out.clone(), idx.clone(), val.clone())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        call()
        torch.cuda.synchronize()
        with torch.cuda.graph(graph, stream=s):
            call()
    torch.cuda.synchronize()
    seen = []
    for n in (counts[0], counts[1], counts[2], counts[1], counts[0]):
        ops.store_i32(dyn, n)
        out.zero_(), idx.zero_(), val.zero_()
        graph.replay()
        _sync()
        st = _stats(ws, K, cap, k)
        assert st[2] == pred[n], (n, st)
        assert all(torch.equal(a, b) for a, b in zip((out, idx, val), want[n])), f"replay at count {n}"
        seen.append(st[2])
    print(f"\ngraph replay, counts {counts}: flagged queries per replay {seen}, each replay the eager bits")


# ------------------------------------------------------------------ workspace hygiene
def test_workspace_contents_do_not_matter(dev):
    """A workspace pre-filled with 0xFF, and one last used by a fallback read of another shape, give the bits of a
    zeroed workspace: top-k, wide and dense reads."""
    L = C.topk_layout("groups", 50, seed=7)
    A = _dev(L["A"], dev)
    K = len(L["live"])
    other = _dev(C.topk_layout("sets", 64, seed=9)["A"], dev)
    W = _dev(C.wide_layout("groups", 256, seed=3)["A"], dev)
    Wo = _dev(C.wide_layout("sets", 1024, seed=4)["A"], dev)
    runs = {
        "top-k": (lambda ws, a=A: ops.memory_read_groups(**a, out=torch.zeros((K, C.HW, 512), device=dev),
                                                         workspace=ws, want_topk=True),
                  lambda ws: ops.memory_read_sets(**other, out=torch.zeros((4, C.HW, 512), device=dev), workspace=ws),
                  max(ops.memory_read_workspace_bytes(K, A["slots"], C.HW, 50),
                      ops.memory_read_workspace_bytes(4, other["slots"], C.HW, 64))),
        "wide": (lambda ws: ops.memory_read_wide_groups(**W, out=torch.zeros((5, C.HW, 512), device=dev),
                                                        workspace=ws, want_topk=True),
                 lambda ws: ops.memory_read_wide_sets(**Wo, out=torch.zeros((4, C.HW, 512), device=dev), workspace=ws),
                 max(ops.memory_read_wide_workspace_bytes(5, W["slots"], C.HW, 256),
                     ops.memory_read_wide_workspace_bytes(4, Wo["slots"], C.HW, 1024))),
        "dense": (lambda ws: (ops.memory_read_dense_groups(A["bank_k"], A["bank_v"], A["slots"], A["qk"],
                                                           torch.zeros((K, C.HW, 512), device=dev), A["counts"],
                                                           A["first"], workspace=ws),),
                  lambda ws: ops.memory_read_dense_sets(other["bank_k"], other["bank_v"], other["slots"], other["qk"],
                                                        torch.zeros((4, C.HW, 512), device=dev), other["counts"],
                                                        workspace=ws),
                  max(ops.memory_read_dense_workspace_bytes(K, A["slots"], C.HW),
                      ops.memory_read_dense_workspace_bytes(4, other["slots"], C.HW))),
    }
    for what, (run, prior, nbytes) in runs.items():
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        want = run(ws)
        _sync()
        ws.fill_(0xFF)
        got_ff = run(ws)
        _sync()
        prior(ws)
        got_prior = run(ws)
        _sync()
        for got, how in ((got_ff, "0xFF"), (got_prior, "a prior read of another shape")):
            assert all(torch.equal(a, b) for a, b in zip(want, got)), f"{what}: workspace left by {how}"
    print("\nworkspaces of 0xFF and of a prior fallback read of another shape: the bits of a zeroed one "
          "(top-k, wide, dense)")


# ------------------------------------------------------------------ cost, reported
def test_fallback_wall_time(dev):
    """Wall time of a grouped top-k read whose objects take the exact fallback against the same launch on a bank
    without the constructions (reported, not asserted)."""
    L = C.topk_layout("groups", 50, seed=7)
    A = _dev(L["A"], dev)
    K = len(L["live"])
    quiet = dict(A, bank_k=A["bank_k"].clone())
    for o in range(K):
        quiet["bank_k"][o, :, :3] = torch.randn((A["slots"], 3), generator=torch.Generator(device=dev).manual_seed(o),
                                                device=dev)
    ws = torch.zeros(ops.memory_read_workspace_bytes(K, A["slots"], C.HW, 50), dtype=torch.uint8, device=dev)
    out = torch.zeros((K, C.HW, 512), device=dev)
    res = {}
    for name, a in (("fallback", A), ("no fallback", quiet)):
        for _ in range(3):
            ops.memory_read_groups(**a, out=out, workspace=ws)
        _sync()
        flagged = _stats(ws, K, A["slots"], 50)[2]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            ops.memory_read_groups(**a, out=out, workspace=ws)
        e1.record()
        _sync()
        res[name] = (e0.elapsed_time(e1) / 20, flagged)
    p = torch.cuda.get_device_properties(0)
    print(f"\n{p.name}: grouped top-50 read, K {K}, hw {C.HW}, counts {L['A']['counts'].tolist()}: "
          + "; ".join(f"{n} {t * 1e3:.0f} us ({f} flagged queries)" for n, (t, f) in res.items()))
