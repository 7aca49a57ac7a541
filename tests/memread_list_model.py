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


if __name__ == "__main__":
    K, frames, top_k = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    mk, qk = features(K, frames)
    run(mk, qk, top_k, bool(int(sys.argv[4])) if len(sys.argv) > 4 else True)
