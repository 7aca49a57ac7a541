// Space-time memory read: EvalMemoryReader.forward + softmax_w_g_top of the reference
// (model/propagation/prop_net.py:47-73, 81-108) without ever materialising the [slots, hw]
// affinity matrix.
//
// Two stages:
//   A. candidate generation over the bank, split over CTAs along the memory axis.  Each
//      (object, query, split) produces a short list of (score, slot) candidates:
//        A1 `memread_exact_kernel`  : fp32 FMA scores on CUDA cores, exact per-split top-k
//                                     (this file; also the overflow fallback of A2)
//        A2 `memread_tc_kernel`     : TF32 wgmma scores + conservative threshold with an error
//                                     margin (memread_tc.cu); survivors are re-scored exactly in B
//   B. `memread_select_kernel`: per (object, query) merge candidates, (re-score,) exact top-k with
//      a total order (score desc, slot asc), softmax over the k survivors
//      (exp(s - s_max) / sum, prop_net.py:55-58), value read-out as a k-row gather of the
//      slot-major value bank (algorithmically 2*k*512 flops/query instead of the reference's
//      dense 2*slots*512).
//
// Score definition (both paths, bit-identical): s = sum_{c=0..127} key[c] * (q[c] / sqrt(128)),
// accumulated with fmaf in ascending channel order; q/sqrt(128) is an IEEE fp32 division exactly
// as `qk / math.sqrt(CK)` at prop_net.py:86.
#include "host_util.h"
#include "pdl.cuh"
#include "memread.h"

#include <cuda_fp16.h>
#include <atomic>

namespace mivos {
extern std::atomic<int64_t> g_launches;

MemreadPlan memread_plan(int k_objects, int64_t slots, int hw, int top_k, int algo) {
  MemreadPlan pl;
  pl.algo = algo;
  if (algo == MIVOS_MEMREAD_TCGEN05) {
    pl.qtile = 128;
    pl.slot_tile = 256;
    pl.kcap = kTcCandCap;
  } else {
    pl.qtile = 32;
    pl.slot_tile = 128;
    pl.kcap = top_k;
  }
  pl.qtiles = ceil_div(hw, pl.qtile);
  const int64_t tiles = ceil_div64(slots, pl.slot_tile);
  // exact path: ~2 CTAs per SM; tensor-core path: ONE wave of CTAs (~200 KB smem = 1 CTA/SM);
  // every split owns at least 4 slot tiles
  const int64_t sms = num_sms();
  int64_t want = algo == MIVOS_MEMREAD_TCGEN05 ? sms / (static_cast<int64_t>(pl.qtiles) * k_objects)
                                               : ceil_div64(2 * sms, static_cast<int64_t>(pl.qtiles) * k_objects);
  int64_t max_by_tiles = tiles / 4 > 0 ? tiles / 4 : 1;
  int64_t s = want < max_by_tiles ? want : max_by_tiles;
  if (s < 1) s = 1;
  if (s > kMaxSplits) s = kMaxSplits;
  pl.tiles_per_split = static_cast<int>(ceil_div64(tiles, s));
  pl.splits = static_cast<int>(ceil_div64(tiles, pl.tiles_per_split));
  pl.nlists = algo == MIVOS_MEMREAD_TCGEN05 ? pl.splits * kTcHalves : pl.splits;
  const int64_t lists = static_cast<int64_t>(k_objects) * hw * pl.nlists;
  pl.off_list = 0;
  pl.off_cnt = lists * pl.kcap * 8 + (algo == MIVOS_MEMREAD_TCGEN05 ? 4096 : 0);  // plan_lists() aligns the lists to 4 KB
  pl.off_flag = 0;  // (overflow flags live in the tail of the workspace: memread_tc_run)
  pl.bytes = pl.off_cnt + lists * 4;
  pl.bytes = (pl.bytes + 255) & ~255ll;
  return pl;
}

namespace {

constexpr float kSqrtCK = 11.313708498984761f;  // sqrt(128) rounded to fp32, as the reference's divisor

constexpr int A1_THREADS = 256;
constexpr int A1_Q = 32;
constexpr int A1_S = 128;
constexpr int KS_STRIDE = 132;  // padded key-row stride (floats): conflict-free LDS.128 by row
constexpr int MAXK = 64;

struct A1Smem {
  float qs[A1_Q][128];
  float ks[A1_S][KS_STRIDE];
  float sc[A1_Q][A1_S + 1];
  float list_s[A1_Q][MAXK];
  int list_i[A1_Q][MAXK];
  float pend_s[A1_Q][A1_S];
  int pend_i[A1_Q][A1_S];
  int pend_cnt[A1_Q];
  int list_cnt[A1_Q];
};

// (score desc, slot asc) total order: true if a ranks before b
__device__ __forceinline__ bool before(float sa, int ia, float sb, int ib) {
  return (sa > sb) || (sa == sb && ia < ib);
}

__global__ void __launch_bounds__(A1_THREADS, 1)
memread_exact_kernel(const float* __restrict__ bank_k, int64_t slots_cap, int64_t slots,
                     const float* __restrict__ qk_all, int hw, int q_div, int top_k, int tiles_per_split,
                     int splits, int2* __restrict__ cand,
                     int* __restrict__ cand_cnt, const int* __restrict__ flags,
                     const int* __restrict__ dyn_slots) {
  mivos::pdl_prologue();
  extern __shared__ __align__(16) uint8_t smem_raw[];
  A1Smem& sm = *reinterpret_cast<A1Smem*>(smem_raw);
  const int tid = threadIdx.x;
  const int q0 = blockIdx.x * A1_Q;
  const int split = blockIdx.y;
  const int obj = blockIdx.z;
  if (flags) {  // fallback mode: only tiles that own an overflowed query do any work
    const int mine = (tid < A1_Q && q0 + tid < hw) ? flags[static_cast<int64_t>(obj) * hw + q0 + tid] : 0;
    if (!__syncthreads_or(mine)) return;
  }
  const float* keys = bank_k + static_cast<int64_t>(obj) * slots_cap * 128;
  const float* qk = qk_all + static_cast<int64_t>(q_div > 0 ? obj / q_div : 0) * hw * 128;  // this object's query set

  // queries, pre-divided by sqrt(CK) (prop_net.py:86)
  for (int i = tid; i < A1_Q * 128; i += A1_THREADS) {
    const int q = i >> 7, c = i & 127;
    sm.qs[q][c] = (q0 + q < hw) ? qk[static_cast<int64_t>(q0 + q) * 128 + c] / kSqrtCK : 0.f;
  }
  if (tid < A1_Q) {
    sm.pend_cnt[tid] = 0;
    sm.list_cnt[tid] = 0;
  }
  __syncthreads();

  if (dyn_slots) {  // device-side slot count (CUDA-graph replay): fixed grid, ranges derived here
    slots = *dyn_slots;
    const int tiles = static_cast<int>((slots + A1_S - 1) / A1_S);
    tiles_per_split = (tiles + splits - 1) / splits;
  }
  const int64_t s_begin = static_cast<int64_t>(split) * tiles_per_split * A1_S;
  int64_t s_end = s_begin + static_cast<int64_t>(tiles_per_split) * A1_S;
  if (s_end > slots) s_end = slots;

  for (int64_t s0 = s_begin; s0 < s_end; s0 += A1_S) {
    // ---- stage 128 key rows (coalesced float4), zero rows past the end
    for (int i = tid; i < A1_S * 32; i += A1_THREADS) {
      const int r = i >> 5, c4 = i & 31;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (s0 + r < s_end) v = *reinterpret_cast<const float4*>(keys + (s0 + r) * 128 + c4 * 4);
      *reinterpret_cast<float4*>(&sm.ks[r][c4 * 4]) = v;
    }
    __syncthreads();
    // ---- 128 slots x 32 queries of fp32 dot products; thread = (slot, 16-query half)
    {
      const int sl = tid & 127, qh = (tid >> 7) * 16;
      float acc[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] = 0.f;
#pragma unroll 4
      for (int c4 = 0; c4 < 32; ++c4) {
        const float4 kv = *reinterpret_cast<const float4*>(&sm.ks[sl][c4 * 4]);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float4 qv = *reinterpret_cast<const float4*>(&sm.qs[qh + j][c4 * 4]);
          acc[j] = fmaf(kv.x, qv.x, acc[j]);
          acc[j] = fmaf(kv.y, qv.y, acc[j]);
          acc[j] = fmaf(kv.z, qv.z, acc[j]);
          acc[j] = fmaf(kv.w, qv.w, acc[j]);
        }
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) sm.sc[qh + j][sl] = acc[j];
    }
    __syncthreads();
    // ---- threshold filter: 8 threads per query, 16 slots each
    {
      const int q = tid >> 3, sub = tid & 7;
      const int cnt = sm.list_cnt[q];
      const float thr = (cnt >= top_k) ? sm.list_s[q][top_k - 1] : -INFINITY;
#pragma unroll 4
      for (int j = 0; j < 16; ++j) {
        const int sl = sub * 16 + j;
        const float s = sm.sc[q][sl];
        if (s0 + sl < s_end && (cnt < top_k || s > thr)) {
          const int pos = atomicAdd(&sm.pend_cnt[q], 1);
          sm.pend_s[q][pos] = s;
          sm.pend_i[q][pos] = static_cast<int>(s0 + sl);
        }
      }
    }
    __syncthreads();
    // ---- merge pending candidates into the sorted per-query list (one thread per query)
    if (tid < A1_Q) {
      const int q = tid;
      int cnt = sm.list_cnt[q];
      const int np = sm.pend_cnt[q];
      for (int p = 0; p < np; ++p) {
        const float s = sm.pend_s[q][p];
        const int id = sm.pend_i[q][p];
        if (cnt == top_k && !before(s, id, sm.list_s[q][cnt - 1], sm.list_i[q][cnt - 1])) continue;
        int pos = (cnt < top_k) ? cnt : cnt - 1;  // slot that will be overwritten / appended
        while (pos > 0 && before(s, id, sm.list_s[q][pos - 1], sm.list_i[q][pos - 1])) {
          sm.list_s[q][pos] = sm.list_s[q][pos - 1];
          sm.list_i[q][pos] = sm.list_i[q][pos - 1];
          --pos;
        }
        sm.list_s[q][pos] = s;
        sm.list_i[q][pos] = id;
        if (cnt < top_k) ++cnt;
      }
      sm.list_cnt[q] = cnt;
      sm.pend_cnt[q] = 0;
    }
    __syncthreads();
  }

  // ---- publish the per-split lists
  for (int i = tid; i < A1_Q * top_k; i += A1_THREADS) {
    const int q = i / top_k, j = i - q * top_k;
    if (q0 + q < hw && j < sm.list_cnt[q]) {
      const int64_t base = ((static_cast<int64_t>(obj) * hw + q0 + q) * splits + split) * top_k;
      cand[base + j] = make_int2(__float_as_int(sm.list_s[q][j]), sm.list_i[q][j]);
    }
  }
  if (tid < A1_Q && q0 + tid < hw)
    cand_cnt[(static_cast<int64_t>(obj) * hw + q0 + tid) * splits + split] = sm.list_cnt[tid];
}

// ------------------------------------------------------------------------------------------
// Stage B.  One WARP per (object, query), kSelWarps queries per CTA.  Everything a query needs —
// gathering its candidate lists, the bisection for a rank-[k, 2k+8] score, compaction, the exact
// re-score, rank counting, softmax and the k-row value gather — is warp-synchronous (shuffles,
// ballots, __syncwarp; no block barrier), so the warps of a CTA are at different phases at any time:
// one query's value gather (k rows of 2 KB from HBM) overlaps another's candidate phase, and
// 3 CTAs x 6 warps stay resident per SM.  (The round-1 kernel ran one query per 128-thread CTA with
// seven block barriers in sequence: 22 % warp occupancy, 47 us at cfg-2 against a ~12 us traffic floor.)
constexpr int kSelWarps = 6;
constexpr int B_THREADS = 32 * kSelWarps;
constexpr int B_MAXSURV = kSelMaxSurvivors;  // candidates (staged) / survivors (re-scored) one query may hold
constexpr int kSelBytesPerWarp = B_MAXSURV * 8 + 128 * 4 + MAXK * 16 + (kMaxLists + 1) * 4 + 28;

__device__ __forceinline__ float exact_score(const float* __restrict__ key, const float* qs) {
  float acc = 0.f;
#pragma unroll 16
  for (int c4 = 0; c4 < 32; ++c4) {
    const float4 kv = *reinterpret_cast<const float4*>(key + c4 * 4);
    acc = fmaf(kv.x, qs[c4 * 4 + 0], acc);
    acc = fmaf(kv.y, qs[c4 * 4 + 1], acc);
    acc = fmaf(kv.z, qs[c4 * 4 + 2], acc);
    acc = fmaf(kv.w, qs[c4 * 4 + 3], acc);
  }
  return acc;
}

struct SelectLists {
  const int2* e;  // {score bits, slot}
  const int* cnt;
  int splits;
  int kcap;
};

__device__ __forceinline__ float warp_min_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__global__ void __launch_bounds__(B_THREADS)
memread_select_kernel(const float* __restrict__ bank_k, const float* __restrict__ bank_v,
                      int64_t slots_cap, const float* __restrict__ qk, int hw, int q_div, int top_k,
                      const SelectLists prim, const int prim_rescore, const SelectLists fb,
                      int* __restrict__ flags, const int pass, const float* __restrict__ qnorm,
                      const float* __restrict__ kmax2, const int* __restrict__ tau_g, void* __restrict__ out, int out_cstride,
                      int out_coff, int halo_h, int halo_w, int out_f16, int* __restrict__ topk_idx,
                      float* __restrict__ topk_val, int* err, const int n_queries) {
  mivos::pdl_prologue();
  extern __shared__ __align__(16) uint8_t sel_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t lq = static_cast<int64_t>(blockIdx.x) * kSelWarps + warp;  // = obj * hw + q
  if (lq >= n_queries) return;
  const int obj = static_cast<int>(lq / hw), q = static_cast<int>(lq - static_cast<int64_t>(obj) * hw);
  const int qset = q_div > 0 ? obj / q_div : 0;  // query set of this object (lock-step clips: one per clip)
  uint8_t* wb = sel_smem + warp * ((kSelBytesPerWarp + 15) & ~15);
  float* cs = reinterpret_cast<float*>(wb);          // [B_MAXSURV] candidate scores
  int* ci = reinterpret_cast<int*>(cs + B_MAXSURV);  // [B_MAXSURV] candidate slots
  float* qs = reinterpret_cast<float*>(ci + B_MAXSURV);  // [128] scaled query
  float* top_s = qs + 128;                           // [MAXK]
  int* top_i = reinterpret_cast<int*>(top_s + MAXK); // [MAXK]
  float* top_w = reinterpret_cast<float*>(top_i + MAXK);  // [MAXK]
  int* order = reinterpret_cast<int*>(top_w + MAXK); // [MAXK]
  int* offs = order + MAXK;                          // [kMaxLists + 1]

  // two-pass protocol (launch_select): pass 0 leaves the flagged queries to pass 1 and may flag more of them below;
  // pass 1 serves the flagged queries only.  Each pass reads ITS lists (`prim`); `fb` is kept for callers that
  // serve both kinds in one launch (none today).
  const bool flagged = flags != nullptr && flags[lq] != 0;
  if (flags != nullptr && (pass == 0) == flagged) return;
  const bool use_fb = false;
  const SelectLists& L = use_fb ? fb : prim;
  const int rescore = prim_rescore;

  // ---- list lengths -> exclusive prefix (the count loads of the lanes are independent)
  {
    const int c = lane < L.splits ? L.cnt[lq * L.splits + lane] : 0;
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    if (lane < L.splits) offs[lane] = incl - c;
    if (lane == L.splits - 1) offs[L.splits] = incl;
  }
  {
    const float4 v = reinterpret_cast<const float4*>(qk + (static_cast<int64_t>(qset) * hw + q) * 128)[lane];
    float4 sq;
    sq.x = v.x / kSqrtCK; sq.y = v.y / kSqrtCK; sq.z = v.z / kSqrtCK; sq.w = v.w / kSqrtCK;
    reinterpret_cast<float4*>(qs)[lane] = sq;
  }
  __syncwarp();
  const int n_all = offs[L.splits];
  // Staging: the concatenated lists are read 128 candidates at a time (four independent loads per lane in flight
  // before the first store) and kept if they pass the generator's FINAL shared threshold minus its margin — every
  // member of the exact top-k does (the lists were written while the threshold was still rising: on cfg-3 features
  // ~1440 candidates per query of which ~380 pass, CPU model in DESIGN.md section 4).  Staging stops when the next
  // chunk might not fit; the rest is filtered from global memory below.
  const float margin = rescore ? kTcMarginFactor * qnorm[static_cast<int64_t>(qset) * hw + q] * sqrtf(kmax2[obj]) : 0.f;
  float cut0 = -INFINITY;
  if (rescore && tau_g) {
    const int o = tau_g[lq];
    cut0 = __int_as_float(o >= 0 ? o : o ^ 0x7fffffff) - margin;
  }
  int n = 0;       // staged candidates
  int i_next = 0;  // first candidate not looked at yet
  {
    int sp = 0;
    for (; i_next < n_all && n + 128 <= B_MAXSURV; i_next += 128) {
      int2 e[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i_next + 32 * u + lane;
        e[u] = make_int2(0, 0);
        if (i < n_all) {
          while (offs[sp + 1] <= i) ++sp;
          e[u] = __ldg(L.e + (lq * L.splits + sp) * L.kcap + (i - offs[sp]));
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i_next + 32 * u + lane;
        const bool keep = i < n_all && __int_as_float(e[u].x) >= cut0;
        const unsigned mask = __ballot_sync(0xffffffffu, keep);
        if (keep) {
          const int pos = n + __popc(mask & ((1u << lane) - 1u));
          cs[pos] = __int_as_float(e[u].x);
          ci[pos] = e[u].y;
        }
        n += __popc(mask);
      }
    }
    if (i_next > n_all) i_next = n_all;
  }
  __syncwarp();

  if (rescore) {
    // The candidate scores are TF32 approximations.  Find a value t whose rank among the STAGED candidates is in
    // [top_k, 2*top_k+8] by bisection (any t with count(>= t) >= top_k over ANY subset of the candidates is a
    // lower bound of the top_k-th largest approximate score), keep the candidates that can still belong to the
    // exact top-k (approx >= t - 2*eps, same margin as the generator) and re-score them with the exact fp32 chain.
    const int kk0 = top_k < n ? top_k : n;
    float lo = INFINITY, hi = -INFINITY;
    for (int i = lane; i < n; i += 32) {
      lo = fminf(lo, cs[i]);
      hi = fmaxf(hi, cs[i]);
    }
    lo = warp_min_f(lo);
    hi = warp_max_f(hi);
    const int limit = 2 * kk0 + 8;
    for (int iter = 0; iter < 26 && n > limit; ++iter) {
      const float mid = 0.5f * lo + 0.5f * hi;
      if (!(mid > lo) || !(mid < hi)) break;  // interval exhausted (ties)
      int c = 0;
      for (int i = lane; i < n; i += 32) c += (cs[i] >= mid) ? 1 : 0;
      c = __reduce_add_sync(0xffffffffu, c);
      if (c >= kk0) {
        lo = mid;
        if (c <= limit) break;
      } else {
        hi = mid;
      }
    }
    const float cut = fmaxf(lo - margin, cut0);
    // in-place compaction of the staged candidates (write index <= read index; a chunk is read by all lanes
    // before any lane writes)
    int m = 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
      const int i = i0 + lane;
      const float sv = i < n ? cs[i] : -INFINITY;
      const int iv = i < n ? ci[i] : 0;
      const bool keep = i < n && sv >= cut;
      const unsigned mask = __ballot_sync(0xffffffffu, keep);
      __syncwarp();
      if (keep) {
        const int pos = m + __popc(mask & ((1u << lane) - 1u));
        cs[pos] = sv;
        ci[pos] = iv;
      }
      m += __popc(mask);
      __syncwarp();
    }
    // candidates beyond the staging capacity (long lists: adversarial near-ties) are filtered against the same
    // cut straight from global memory
    bool too_many = false;
    if (n_all > i_next) {
      int sp = 0;
      for (int i0 = i_next; i0 < n_all; i0 += 32) {
        const int i = i0 + lane;
        int2 e = make_int2(0, 0);
        if (i < n_all) {
          while (offs[sp + 1] <= i) ++sp;
          e = L.e[(lq * L.splits + sp) * L.kcap + (i - offs[sp])];
        }
        const bool keep = i < n_all && __int_as_float(e.x) >= cut;
        const unsigned mask = __ballot_sync(0xffffffffu, keep);
        const int pos = m + __popc(mask & ((1u << lane) - 1u));
        if (keep && pos < B_MAXSURV) ci[pos] = e.y;
        m += __popc(mask);
      }
      __syncwarp();
    }
    if (m > B_MAXSURV) {  // more than 1024 candidates within the TF32 margin of the top-k
      too_many = true;
      m = B_MAXSURV;
    }
    if (too_many) {
      // more in-band candidates than this stage can re-score (a margin of the order of the score spread: huge-norm
      // keys): with the two-pass protocol the query goes to the exact CUDA-core generator and pass 1 (m is
      // warp-uniform: the whole warp leaves); without it there is nobody to hand it to
      if (flags != nullptr && pass == 0) {
        if (lane == 0) flags[lq] = 1;
        return;
      }
      if (lane == 0 && err) atomicExch(err, 202);
    }
    n = m;
    // exact fp32 scores, one survivor per lane per pass (normally two passes: n ~ 2k + margin hits)
    const float* keys = bank_k + static_cast<int64_t>(obj) * slots_cap * 128;
    for (int i = lane; i < n; i += 32) cs[i] = exact_score(keys + static_cast<int64_t>(ci[i]) * 128, qs);
    __syncwarp();
  } else if (n_all > i_next) {  // cannot happen: exact lists hold top_k entries per split
    if (lane == 0 && err) atomicExch(err, 201);
  }

  // ---- exact top-k by rank counting under the (score desc, slot asc) total order
  const int kk = top_k < n ? top_k : n;
  for (int i = lane; i < n; i += 32) {
    const float si = cs[i];
    const int ii = ci[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) rank += before(cs[j], ci[j], si, ii) ? 1 : 0;
    if (rank < kk) {
      top_s[rank] = si;
      top_i[rank] = ii;
    }
  }
  __syncwarp();
  // ---- softmax over the survivors: exp(s - s_0) / sum (prop_net.py:55-58)
  for (int j = lane; j < kk; j += 32) top_w[j] = expf(top_s[j] - top_s[0]);
  __syncwarp();
  float sum = 0.f;
  for (int j = 0; j < kk; ++j) sum += top_w[j];  // same sequential sum in every lane
  // accumulation order of the read-out: ascending slot index
  for (int t = lane; t < kk; t += 32) {
    int r = 0;
    for (int j = 0; j < kk; ++j) r += (top_i[j] < top_i[t]) ? 1 : 0;
    order[r] = t;
  }
  __syncwarp();
  if (topk_idx)
    for (int t = lane; t < top_k; t += 32) topk_idx[lq * top_k + t] = t < kk ? top_i[t] : -1;
  if (topk_val)
    for (int t = lane; t < top_k; t += 32) topk_val[lq * top_k + t] = t < kk ? top_s[t] : 0.f;

  // ---- read-out: the lane owns float4 pieces lane, lane+32, lane+64, lane+96 of the 512 value channels
  float4 acc[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4* vals = reinterpret_cast<const float4*>(bank_v + static_cast<int64_t>(obj) * slots_cap * 512);
  // rows in batches of 4 (16 independent 16-byte loads per lane in flight); the accumulation order per channel
  // stays ascending slot index
  for (int j0 = 0; j0 < kk; j0 += 4) {
    float4 v[4][4];
    float w[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int jj = j0 + r;
      const int j = order[jj < kk ? jj : kk - 1];
      w[r] = top_w[j] / sum;
      const float4* row = vals + static_cast<int64_t>(top_i[j]) * 128;
#pragma unroll
      for (int u = 0; u < 4; ++u) v[r][u] = row[lane + 32 * u];
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      if (j0 + r < kk) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          acc[u].x = fmaf(w[r], v[r][u].x, acc[u].x);
          acc[u].y = fmaf(w[r], v[r][u].y, acc[u].y);
          acc[u].z = fmaf(w[r], v[r][u].z, acc[u].z);
          acc[u].w = fmaf(w[r], v[r][u].w, acc[u].w);
        }
      }
    }
  }
  int64_t row;
  if (halo_w > 0) {
    const int y = q / halo_w, x = q - y * halo_w;
    row = (static_cast<int64_t>(obj) * (halo_h + 2) + y + 1) * (halo_w + 2) + x + 1;
  } else {
    row = lq;
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int c = (lane + 32 * u) * 4;
    if (out_f16) {
      const __half2 h01 = __floats2half2_rn(acc[u].x, acc[u].y), h23 = __floats2half2_rn(acc[u].z, acc[u].w);
      uint2 pk;
      pk.x = *reinterpret_cast<const uint32_t*>(&h01);
      pk.y = *reinterpret_cast<const uint32_t*>(&h23);
      *reinterpret_cast<uint2*>(static_cast<__half*>(out) + row * out_cstride + out_coff + c) = pk;
    } else {
      *reinterpret_cast<float4*>(static_cast<float*>(out) + row * out_cstride + out_coff + c) = acc[u];
    }
  }
}

}  // namespace

int launch_exact_candidates(const float* bank_k, int64_t slots_cap, int k_objects, int64_t slots,
                            const float* qk, int hw, int q_div, int top_k, const MemreadPlan& pl, void* ws,
                            const int* flags, const int* dyn_slots, cudaStream_t stream) {
  static bool configured = false;
  if (!configured) {
    MIVOS_CUDA_OK(cudaFuncSetAttribute(memread_exact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(sizeof(A1Smem))));
    configured = true;
  }
  uint8_t* w = static_cast<uint8_t*>(ws);
  dim3 grid(pl.qtiles, pl.splits, k_objects);
  launch_pdl(memread_exact_kernel, grid, A1_THREADS, sizeof(A1Smem), stream, 
      bank_k, slots_cap, slots, qk, hw, q_div, top_k, pl.tiles_per_split, pl.splits,
      reinterpret_cast<int2*>(plan_lists(w, pl)),
      reinterpret_cast<int*>(w + pl.off_cnt), flags, dyn_slots);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  MIVOS_CUDA_OK(cudaGetLastError());
  return MIVOS_OK;
}

int launch_select(const float* bank_k, const float* bank_v, int64_t slots_cap, int k_objects,
                  const float* qk, int hw, int q_div, int top_k, const MemreadPlan& pl, void* ws,
                  const MemreadPlan* fbp, void* fb_ws, int* flags, int pass, const float* qnorm,
                  const float* kmax2, const int* tau_g, void* out, int out_cstride, int out_coff, int halo_h,
                  int halo_w, int out_f16, int32_t* topk_idx, float* topk_val, cudaStream_t stream) {
  uint8_t* w = static_cast<uint8_t*>(ws);
  SelectLists prim{reinterpret_cast<const int2*>(plan_lists(w, pl)), reinterpret_cast<const int*>(w + pl.off_cnt),
                   pl.nlists, pl.kcap};
  SelectLists fb = prim;
  if (fbp) {
    uint8_t* f = static_cast<uint8_t*>(fb_ws);
    fb = SelectLists{reinterpret_cast<const int2*>(plan_lists(f, *fbp)), reinterpret_cast<const int*>(f + fbp->off_cnt),
                     fbp->nlists, fbp->kcap};
  }
  const int rescore = pl.algo == MIVOS_MEMREAD_TCGEN05 ? 1 : 0;
  MIVOS_REQUIRE(prim.splits <= 32 && fb.splits <= 32, "memory_read: more than 32 candidate lists per query");
  constexpr int smem = kSelWarps * ((kSelBytesPerWarp + 15) & ~15);
  static bool configured = false;
  if (!configured) {
    MIVOS_CUDA_OK(cudaFuncSetAttribute(memread_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  const int n_queries = k_objects * hw;
  dim3 grid(ceil_div(n_queries, kSelWarps));
  launch_pdl(memread_select_kernel, grid, B_THREADS, smem, stream, bank_k, bank_v, slots_cap, qk, hw, q_div, top_k, prim, rescore, fb,
                                                           flags, pass, qnorm, kmax2, tau_g, out, out_cstride,
                                                           out_coff, halo_h, halo_w, out_f16, topk_idx, topk_val,
                                                           device_error_flag(), n_queries);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  MIVOS_CUDA_OK(cudaGetLastError());
  return MIVOS_OK;
}

}  // namespace mivos

using namespace mivos;

// tail of the workspace after the two plans' lists: flags [K*hw] | key-norm maxima [kMaxObjects] | scaled queries
// [K*hw*128] (one set per object at most) | their norms [K*hw, padded to 64] | shared thresholds [K*hw]
static int64_t memread_tail_bytes(int k_objects, int hw) {
  const int64_t nq = static_cast<int64_t>(k_objects) * hw, nq64 = (nq + 63) & ~63ll;
  return (nq64 + kMaxObjects + nq * 128 + nq64 + nq64) * 4 + 1024;
}

extern "C" MIVOS_API int64_t mivos_memory_read_workspace(int k_objects, int64_t slots, int hw, int top_k) {
  if (k_objects < 1 || k_objects > kMaxObjects || slots < 1 || hw < 1 || top_k < 1 || top_k > MAXK) return -1;
  const MemreadPlan a = memread_plan(k_objects, slots, hw, top_k, MIVOS_MEMREAD_EXACT_SIMT);
  const MemreadPlan b = memread_plan(k_objects, slots, hw, top_k, MIVOS_MEMREAD_TCGEN05);
  return b.bytes + a.bytes + memread_tail_bytes(k_objects, hw);
}

extern "C" MIVOS_API int mivos_memory_read(const float* bank_k, const float* bank_v, int64_t slots_cap,
                                           int k_objects, int64_t slots, const float* qk, int hw, int q_div,
                                           int top_k, void* out, int out_cstride, int out_coff,
                                           int out_halo_h, int out_halo_w, int32_t* topk_idx,
                                           float* topk_val, void* workspace, int64_t workspace_bytes,
                                           int algo, const int32_t* dyn_slots, int out_f16, mivos_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MIVOS_REQUIRE(bank_k && bank_v && qk && out && workspace, "memory_read: null pointer");
  MIVOS_REQUIRE(top_k >= 1 && top_k <= MAXK, "memory_read: top_k %d outside [1,%d]", top_k, MAXK);
  MIVOS_REQUIRE(slots >= top_k && slots <= slots_cap && slots < (1ll << 31) - 65536,
                "memory_read: bad slot count %lld (cap %lld, k %d)", (long long)slots, (long long)slots_cap, top_k);
  MIVOS_REQUIRE(k_objects >= 1 && k_objects <= kMaxObjects && hw >= 1, "memory_read: bad object/query count");
  MIVOS_REQUIRE(q_div >= 0, "memory_read: q_div must be >= 0 (0: all objects read one query set)");
  MIVOS_REQUIRE(out_cstride % 4 == 0 && out_coff % 4 == 0 && out_coff + 512 <= out_cstride,
                "memory_read: output channel window does not fit");
  MIVOS_REQUIRE(out_halo_w == 0 || out_halo_h * out_halo_w == hw, "memory_read: halo dims do not match hw");
  MIVOS_REQUIRE((reinterpret_cast<uintptr_t>(bank_k) & 15) == 0 && (reinterpret_cast<uintptr_t>(bank_v) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0,
                "memory_read: pointers must be 16-byte aligned (workspace 256)");
  const int64_t need = mivos_memory_read_workspace(k_objects, slots, hw, top_k);
  MIVOS_REQUIRE(workspace_bytes >= need, "memory_read: workspace %lld < %lld bytes", (long long)workspace_bytes, (long long)need);
  if (algo == MIVOS_MEMREAD_AUTO) algo = memread_tc_available() ? MIVOS_MEMREAD_TCGEN05 : MIVOS_MEMREAD_EXACT_SIMT;

  if (algo == MIVOS_MEMREAD_EXACT_SIMT) {
    const MemreadPlan pl = memread_plan(k_objects, slots, hw, top_k, MIVOS_MEMREAD_EXACT_SIMT);
    int rc = launch_exact_candidates(bank_k, slots_cap, k_objects, slots, qk, hw, q_div, top_k, pl, workspace, nullptr, dyn_slots, stream);
    if (rc != MIVOS_OK) return rc;
    return launch_select(bank_k, bank_v, slots_cap, k_objects, qk, hw, q_div, top_k, pl, workspace, nullptr, nullptr,
                         nullptr, 0, nullptr, nullptr, nullptr, out, out_cstride, out_coff, out_halo_h, out_halo_w, out_f16, topk_idx,
                         topk_val, stream);
  }
  if (algo == MIVOS_MEMREAD_TCGEN05) {
    return memread_tc_run(bank_k, bank_v, slots_cap, k_objects, slots, qk, hw, q_div, top_k, out, out_cstride,
                          out_coff, out_halo_h, out_halo_w, out_f16, topk_idx, topk_val, workspace, dyn_slots, stream);
  }
  set_last_error("memory_read: unknown algo %d", algo);
  return MIVOS_ERR_INVALID;
}

// Debug/diagnostic (synchronises): candidate statistics of the last tensor-core-path read that used
// `workspace`: out[0] = total candidates after compaction, out[1] = max per (object, query),
// out[2] = queries flagged for the exact fallback, out[3] = splits.
extern "C" MIVOS_API int mivos_memory_read_stats(const void* workspace, int k_objects, int64_t slots, int hw,
                                                 int top_k, int64_t* out) {
  MIVOS_REQUIRE(workspace && out, "memory_read_stats: null pointer");
  const MemreadPlan tc = memread_plan(k_objects, slots, hw, top_k, MIVOS_MEMREAD_TCGEN05);
  const MemreadPlan ex = memread_plan(k_objects, slots, hw, top_k, MIVOS_MEMREAD_EXACT_SIMT);
  const int64_t nq = static_cast<int64_t>(k_objects) * hw;
  int* cnt = new int[nq * tc.nlists];
  int* flg = new int[nq];
  const uint8_t* w = static_cast<const uint8_t*>(workspace);
  cudaError_t e1 = cudaMemcpy(cnt, w + tc.off_cnt, nq * tc.nlists * 4, cudaMemcpyDeviceToHost);
  cudaError_t e2 = cudaMemcpy(flg, w + tc.bytes + ex.bytes, nq * 4, cudaMemcpyDeviceToHost);
  int64_t total = 0, mx = 0, flagged = 0;
  if (e1 == cudaSuccess && e2 == cudaSuccess) {
    for (int64_t q = 0; q < nq; ++q) {
      int64_t s = 0;
      if (flg[q]) { ++flagged; continue; }
      for (int sp = 0; sp < tc.nlists; ++sp) s += cnt[q * tc.nlists + sp];
      total += s;
      if (s > mx) mx = s;
    }
  }
  delete[] cnt;
  delete[] flg;
  MIVOS_CUDA_OK(e1);
  MIVOS_CUDA_OK(e2);
  out[0] = total; out[1] = mx; out[2] = flagged; out[3] = tc.splits;
  return MIVOS_OK;
}
