"""CPU: the premises and the teeth of tests/test_gpu_memread_fallback.py.

Premises: on the banks of tests/memread_fallback_cases.py, the model of tests/memread_list_model.py shows that each
construction takes exactly its branch with slack — at least 1.5x above, or at most 0.5x below, each threshold it is
meant to cross or not (384 per list while streaming, 1024 survivors in pass A, 896 staged candidates), so the TF32
rounding on the GPU cannot move a designed query across — and that every other query stays at most 0.5x below both
flag thresholds under every timing and rounding (`high_tf32`, `survivors_max`).  The wide read's constructions give the intended modes on their exact fp32 scores.

Teeth: a host emulation of the top-k read's two-pass protocol (flags from the model, flagged queries served by the
exact fallback) passes `memory_census.checked_read` and the strict tie check on random banks and on the new cases,
and each of these bugs, harmless on random banks, fails the new cases: pass B serving a flagged query with group 0's
count and query set; pass B serving it with group 0's query set and its own count (the designed queries of set g are
scaled by 2^g, so the indices stay and the scores and read-out change); selection-flagged queries never served, so
the sentinel survives; the exact fallback tile serving only its first flagged query."""
import math

import numpy as np
import pytest
import torch

import memory_census as MC
import memread_fallback_cases as C
import memread_list_model as LM


# ------------------------------------------------------------------ premises
@pytest.mark.parametrize("form", ["qdiv", "scalar", "sets", "groups"])
@pytest.mark.parametrize("k", [20, 50, 64])
def test_constructions_take_their_branch_with_slack(form, k):
    L = C.topk_layout(form, k, seed=7)
    flags = 0
    for o, m in enumerate(C.model_flags(L)):
        designs = L["designs"][o]
        for q in range(C.HW):
            role = C.TOPK_ROLES.get(q, "quiet")
            where = f"{form} k {k} object {o} query {q} ({role})"
            lists_high, lists_low = int(m["high_tf32"][q].max()), int(m["low"][q].max())
            if role in designs and role == "stream":
                assert lists_low >= 1.5 * LM.LIST_LIMIT, where
            elif role in designs:
                assert lists_high <= 0.5 * LM.LIST_LIMIT, where
                if role == "select":
                    assert m["band"][q] >= 1.5 * LM.SEL_CAP, where
                else:
                    assert m["staged"][q] >= 1.5 * LM.STAGE_LIMIT, where
                    assert m["survivors"][q] <= 0.5 * LM.SEL_CAP, where
                    # the k largest sit in the first two lists, which staging always reads whole
                    keys = L["A"]["bank_k"][o, :L["live"][o], C.CH_GLOBAL].numpy()
                    top = np.argsort(-keys, kind="stable")[:k]
                    assert (top // LM.TS < L["tps"][o]).all(), where
            else:
                # not a construction (quiet, or its channel holds no construction in this object)
                assert lists_high <= 0.5 * LM.LIST_LIMIT and m["survivors_max"][q] <= 0.5 * LM.SEL_CAP, where
            flags += int(m["flag"][q])
    assert flags == C.predicted_flags(L) and 0 < flags < len(L["live"]) * C.HW


def test_lists_model_bounds_a_plain_bank():
    """On N(0, 1) data the lower and upper list bounds bracket each other and nothing flags."""
    g = np.random.default_rng(0)
    keys = g.standard_normal((8000, 128)).astype(np.float32)
    qs = (g.standard_normal((40, 128)) / math.sqrt(128)).astype(np.float32)
    splits, tps = LM.tc_plan(8000, 1, 40, 132)
    m = LM.read_model(keys, qs, 20, splits, tps)
    assert (m["low"] <= np.maximum(m["high"], LM.LIST_LIMIT)).all()
    assert not m["flag"].any() and (m["survivors"] <= m["survivors_max"]).all()
    exact = -np.sort(-(qs.astype(np.float64) @ keys.T.astype(np.float64)), 1)[:, 19]
    assert (m["tau_g"] <= exact + 1e-3).all()


@pytest.mark.parametrize("k", [65, 256, 1024])
def test_wide_constructions_give_their_modes(k):
    L = C.wide_layout("groups", k, seed=3)
    want = {0: (0, False), 1: (0, True), 2: (2, True), 3: (2, True), 4: (0, False)}
    keys = L["A"]["bank_k"]
    for o, n in enumerate(L["live"]):
        if not L["designed"][o]:
            continue
        for c, mode in want.items():
            col = keys[o, :n, c].numpy()
            assert LM.wide_state(col, k) == mode, (o, c)
            kth = np.sort(col)[::-1][k - 1]
            u = LM.score_key(col)
            if c == 2:  # > 2048 distinct scores in the k-th score's level-2 bin
                same_bin = (u >> 14) == (LM.score_key(np.float32([kth]))[0] >> 14)
                assert np.unique(col[same_bin]).size > LM.WIDE_CAP
            if c in (3, 4):  # bit-identical rows straddle rank k
                srt = np.sort(col)[::-1]
                assert srt[k - 2] == srt[k - 1] == srt[k] == C.LEVEL
    modes = {m for row in C.wide_predicted(L) for m in row}
    assert {(0, False), (0, True), (2, True)} <= modes


# ------------------------------------------------------------------ teeth
def _fallback_read(mutate, sms=132):
    """memory_read_groups on the host: unflagged queries get the exact (score desc, slot asc) top-k of their fp32
    scores, flagged ones (flags from the list model) are served by an emulated pass B that `mutate` may break."""
    memo = {}

    def kernel(bank_k, bank_v, slots, qk, top_k, out, counts, first, *, out_coff=0, halo_hw=None, workspace=None,
               algo=0, want_topk=False):
        f = [int(v) for v in first]
        cnt = [int(v) for v in counts]
        K = bank_k.shape[0]
        splits, tps = LM.tc_plan(slots, K, qk.shape[1], sms)
        hw = qk.shape[1]
        idx_all = torch.full((K, hw, top_k), -1, dtype=torch.int32)
        val_all = torch.zeros((K, hw, top_k))

        def serve(o, n, q, qrows):
            s = (bank_k[o, :n] @ (q[qrows] / np.float32(math.sqrt(128))).t()).t()       # [c, n] fp32
            order = np.lexsort((np.broadcast_to(np.arange(n), s.shape), -s.double().numpy()), axis=1)[:, :top_k]
            idx = torch.from_numpy(order)
            vals = s.gather(1, idx)
            w = torch.softmax(vals.double(), 1)
            rows = torch.einsum("ck,ckd->cd", w, bank_v[o][idx].double()).float()
            if halo_hw is not None:
                for j, qq in enumerate(qrows.tolist()):
                    out[o, 1 + qq // halo_hw[1], 1 + qq % halo_hw[1], out_coff:out_coff + 512] = rows[j].to(out.dtype)
            else:
                out[o, qrows, out_coff:out_coff + 512] = rows.to(out.dtype)
            idx_all[o, qrows] = idx.int()
            val_all[o, qrows] = vals

        for g in range(len(f) - 1):
            for o in range(f[g], f[g + 1]):
                n = cnt[g]
                key = (id(bank_k), o, n, g)
                if key not in memo:
                    qs = (qk[g].numpy() / C.SQ).astype(np.float32)
                    m = LM.read_model(bank_k[o, :n].numpy(), qs, top_k, splits, LM.live_tps(n, splits, tps, True))
                    memo[key] = (m["flag"], m["select_flag"])
                flag, sel = memo[key]
                plain = torch.from_numpy(np.flatnonzero(~flag))
                if plain.numel():
                    serve(o, n, qk[g], plain)
                served = mutate(flag, sel)
                if served.any():
                    gb, nb = mutate.group(g, n, cnt)
                    serve(o, nb, qk[gb], torch.from_numpy(np.flatnonzero(served)))
        return (out, idx_all, val_all) if want_topk else out
    return kernel


class _Correct:
    def __call__(self, flag, sel):
        return flag

    def group(self, g, n, cnt):
        return g, n


class _GroupZero(_Correct):
    def group(self, g, n, cnt):
        return 0, cnt[0]


class _QuerySetZero(_Correct):
    """Pass B reads query set 0 with the object's own count."""
    def group(self, g, n, cnt):
        return 0, n


class _SelectNeverServed(_Correct):
    def __call__(self, flag, sel):
        return flag & ~sel


class _FirstOfTileOnly(_Correct):
    def __call__(self, flag, sel):
        out = np.zeros_like(flag)
        for t0 in range(0, flag.size, 32):
            hit = np.flatnonzero(flag[t0:t0 + 32])
            if hit.size:
                out[t0 + hit[0]] = True
        return out


def _random_groups(k):
    """A random grouped launch: no query flags."""
    g = torch.Generator().manual_seed(5)
    sizes, counts = [1, 2, 1], [1500, 1201, 1333]
    K = sum(sizes)
    return dict(bank_k=torch.randn((K, 1600, 128), generator=g), bank_v=torch.randn((K, 1600, 512), generator=g),
                slots=1600, qk=torch.randn((3, C.HW, 128), generator=g), top_k=k,
                counts=torch.tensor(counts, dtype=torch.int32), first=torch.tensor([0, 1, 3, 4], dtype=torch.int32),
                out=torch.full((K, C.HW, 640), -3.5), out_coff=64)


@pytest.fixture(scope="module")
def fallback_case():
    L = C.topk_layout("groups", 20, seed=7)
    A = dict(L["A"], out=torch.full((len(L["live"]), C.H + 2, C.W + 2, 1024), -3.5), out_coff=256, halo_hw=(C.H, C.W))
    return L, A


def _fresh(A):
    return dict(A, out=torch.full_like(A["out"], -3.5))


MUTANTS = [(_GroupZero(), "another top-20 set|outside \\[0|exceeds the bound"),
           (_QuerySetZero(), "another top-20 set|exceeds the bound"),
           (_SelectNeverServed(), "outside \\[0|exceeds the bound"),   # no index written, the sentinel survives
           (_FirstOfTileOnly(), "outside \\[0|exceeds the bound")]


def test_emulated_fallback_passes(fallback_case):
    L, A = fallback_case
    rec = MC.checked_read("memory_read_groups", _fallback_read(_Correct()), _fresh(A))
    assert rec["ratio"] <= 1.0
    _, idx, val = _fallback_read(_Correct())(**_fresh(A), want_topk=True)
    C.strict_check(A, L["live"], L["qset"], idx, val,
                   lambda o: C.topk_scores(A["bank_k"][o, :L["live"][o]], L["qset"][o]))


@pytest.mark.parametrize("mutant,match", MUTANTS, ids=["pass_b_with_group_0", "pass_b_with_query_set_0",
                                                       "select_flags_never_served",
                                                       "first_flagged_of_tile_only"])
def test_fallback_bugs_pass_random_banks_and_fail_the_new_cases(fallback_case, mutant, match):
    A = _random_groups(20)
    assert MC.checked_read("memory_read_groups", _fallback_read(mutant), A)["ratio"] <= 1.0
    _, A = fallback_case
    with pytest.raises(AssertionError, match=match):
        MC.checked_read("memory_read_groups", _fallback_read(mutant), _fresh(A))
