// Wide top-k memory read: EvalMemoryReader(top_k=k) for 1 <= k <= 1024 (model/propagation/prop_net.py:47-73, 81-108),
// the same semantics as the top-k read of memread.cu (which holds k <= 64 in registers and warp-sized buffers).
//
// Every score is the exact fp32 chain of `exact_score` (memread.h), computed by a tiled CUDA-core GEMM, so the
// threshold is exact and no error margin is needed.  The selection key of a score is its order-preserving unsigned
// encoding u = float_ordered(s) ^ 0x80000000 (a score is never -0, so u orders exactly as the float compare does).
//
//   1. level-1 sweep   `memread_wide_sweep_kernel<0>`: per-query histogram of the top 9 bits of u (sign, exponent),
//                      in shared memory per CTA, merged over the splits of the memory axis with global atomics.
//   2. `memread_wide_threshold_kernel<0>`: the bin d1 holding the k-th largest score.  If every slot in bins >= d1
//                      fits a query's candidate region (kWideCap), the cut is d1; otherwise the query is refined.
//   3. level-2 sweep   (refined queries only; CTAs without one exit at once): histogram of bits 14..22 of the
//                      scores in bin d1, and `memread_wide_threshold_kernel<1>`: the cut (d1, d2).  A query whose
//                      band still exceeds kWideCap (ties or near-ties over ~2^-9 relative width) is marked for the
//                      exact fallback before anything is emitted, so no candidate list is ever truncated.
//   4. emission sweep  `memread_wide_sweep_kernel<2>`: every (score, slot) with u >= cut into the query's region.
//   5. `memread_wide_select_kernel`, one CTA per (object, query): sort the candidates under the total order (score
//                      desc, slot asc), softmax over the first k (exp(s - s_0) / sum, the sum sequential in rank
//                      order), read-out in ascending slot order, store with `store_read_row`.  A marked query is served
//                      in the same CTA by a radix select over u (4 x 8 bits) of every live slot, re-scored per pass.
// The rank-order sum and the slot-order FMA chain are those of memread_select_kernel, so for k <= 64 this read gives
// the same bits as mivos_memory_read.  Emission order is not deterministic; the sort makes the result so.
#include "host_util.h"
#include "pdl.cuh"
#include "memread.h"

#include <atomic>
#include <cstddef>

namespace mivos {
extern std::atomic<int64_t> g_launches;

namespace {

constexpr int kWideMaxK = 1024;
constexpr int kWideCap = 2048;  // candidates one (object, query) may hold; >= 2 * kWideMaxK
constexpr int kBins = 512;      // 9-bit digits of u
constexpr int kShift1 = 23;     // level-1 digit: u >> 23
constexpr int kShift2 = 14;     // level-2 digit: (u >> 14) & 511

constexpr int WQ = 64;   // queries per sweep CTA
constexpr int WS = 128;  // slots per tile
constexpr int WC = 32;   // channels per staged key chunk
constexpr int W_THREADS = 256;  // thread = 4 queries x 8 slots of the tile

// Per-query state between the launches.  mode 0: emit u >= cut; 1: refine inside level-1 bin d1 (`above` slots rank
// above that bin); 2: exact fallback.
struct WideState {
  unsigned cut;
  int d1;
  int above;
  int mode;
};

struct SweepSmem {
  float qT[128][WQ + 4];  // scaled queries, channel-major
  float kT[WC][WS + 4];   // key chunk, channel-major
  unsigned cut[WQ];
  int d1[WQ];
  int on[WQ];             // the query takes part in this sweep
  unsigned hist[WQ][kBins];  // histogram sweeps only (the emission sweep is launched without it)
};

__device__ __forceinline__ unsigned score_key(float s) { return static_cast<unsigned>(float_ordered(s)) ^ 0x80000000u; }

template <int LEVEL>  // 0: level-1 histogram, 1: level-2 histogram, 2: emission
__global__ void __launch_bounds__(W_THREADS, 1)
memread_wide_sweep_kernel(const MemreadArgs a, const int splits, const WideState* __restrict__ state,
                          unsigned* __restrict__ hist_g, int2* __restrict__ cand, int* __restrict__ cand_cnt) {
  mivos::pdl_prologue();
  extern __shared__ __align__(16) uint8_t smem_raw[];
  SweepSmem& sm = *reinterpret_cast<SweepSmem*>(smem_raw);
  const int tid = threadIdx.x;
  const int hw = a.hw;
  const int q0 = blockIdx.x * WQ, split = blockIdx.y, obj = blockIdx.z;
  const int nq = hw - q0 < WQ ? hw - q0 : WQ;
  const int64_t lq0 = static_cast<int64_t>(obj) * hw + q0;

  int part = 0;
  if (tid < WQ) {
    WideState s{0u, 0, 0, 0};
    if (tid < nq) {
      if (LEVEL > 0) s = state[lq0 + tid];
      part = LEVEL == 0 ? 1 : (LEVEL == 1 ? s.mode == 1 : s.mode == 0);
    }
    sm.cut[tid] = s.cut;
    sm.d1[tid] = s.d1;
    sm.on[tid] = part;
  }
  if (!__syncthreads_or(part)) return;

  if (LEVEL < 2)
    for (int i = tid; i < WQ * kBins; i += W_THREADS) (&sm.hist[0][0])[i] = 0u;
  const int qset = query_set(a, obj);
  const float* qk = a.qk + (static_cast<int64_t>(qset) * hw + q0) * 128;
  for (int i = tid; i < WQ * 128; i += W_THREADS) {
    const int q = i >> 7, c = i & 127;
    sm.qT[c][q] = q < nq ? qk[static_cast<int64_t>(q) * 128 + c] / kSqrtCK : 0.f;  // prop_net.py:86
  }

  const int64_t live = live_slots(a, obj);
  const int64_t tiles = (live + WS - 1) / WS;
  const float* keys = a.bank_k + static_cast<int64_t>(obj) * a.slots_cap * 128;
  const int tq = tid & 15, ts = tid >> 4;
  for (int64_t t = split; t < tiles; t += splits) {
    const int64_t s0 = t * WS;
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    for (int c0 = 0; c0 < 128; c0 += WC) {
      __syncthreads();  // the previous chunk has been consumed (and, first time round, qT / hist are ready)
      for (int i = tid; i < WS * WC / 4; i += W_THREADS) {
        const int r = i & (WS - 1), j = i >> 7;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (s0 + r < live) v = *reinterpret_cast<const float4*>(keys + (s0 + r) * 128 + c0 + 4 * j);
        sm.kT[4 * j + 0][r] = v.x;
        sm.kT[4 * j + 1][r] = v.y;
        sm.kT[4 * j + 2][r] = v.z;
        sm.kT[4 * j + 3][r] = v.w;
      }
      __syncthreads();
#pragma unroll 4
      for (int c = 0; c < WC; ++c) {
        const float4 qv = *reinterpret_cast<const float4*>(&sm.qT[c0 + c][tq * 4]);
        const float4 k0 = *reinterpret_cast<const float4*>(&sm.kT[c][ts * 8]);
        const float4 k1 = *reinterpret_cast<const float4*>(&sm.kT[c][ts * 8 + 4]);
        const float qa[4] = {qv.x, qv.y, qv.z, qv.w};
        const float kb[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(kb[j], qa[i], acc[i][j]);  // exact_score's chain
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int ql = tq * 4 + i;
      if (!sm.on[ql]) continue;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int64_t slot = s0 + ts * 8 + j;
        if (slot >= live) continue;
        const unsigned u = score_key(acc[i][j]);
        if (LEVEL == 0) {
          atomicAdd(&sm.hist[ql][u >> kShift1], 1u);
        } else if (LEVEL == 1) {
          if (static_cast<int>(u >> kShift1) == sm.d1[ql]) atomicAdd(&sm.hist[ql][(u >> kShift2) & (kBins - 1)], 1u);
        } else if (u >= sm.cut[ql]) {
          const int64_t lq = lq0 + ql;
          const int pos = atomicAdd(cand_cnt + lq, 1);
          if (pos < kWideCap) cand[lq * kWideCap + pos] = make_int2(__float_as_int(acc[i][j]), static_cast<int>(slot));
        }
      }
    }
  }
  if (LEVEL < 2) {
    __syncthreads();
    for (int i = tid; i < nq * kBins; i += W_THREADS) {
      const int q = i / kBins;
      const unsigned h = (&sm.hist[0][0])[i];
      if (sm.on[q] && h) atomicAdd(hist_g + lq0 * kBins + i, h);
    }
  }
}

// One warp per (object, query): the bin of the level's histogram that holds rank `top_k - above` from the top.
template <int LEVEL>
__global__ void __launch_bounds__(256)
memread_wide_threshold_kernel(const int64_t nq, const int top_k, WideState* __restrict__ state,
                              unsigned* __restrict__ hist_g) {
  mivos::pdl_prologue();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t lq = static_cast<int64_t>(blockIdx.x) * 8 + warp;
  if (lq >= nq) return;
  WideState s{0u, 0, 0, 0};
  if (LEVEL == 1) {
    s = state[lq];
    if (s.mode != 1) return;
  }
  uint4* row = reinterpret_cast<uint4*>(hist_g + lq * kBins) + lane * 4;  // the lane's bins 16 * lane ...
  unsigned c[16];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const uint4 v = row[u];
    c[4 * u] = v.x; c[4 * u + 1] = v.y; c[4 * u + 2] = v.z; c[4 * u + 3] = v.w;
  }
  if (LEVEL == 0)  // the level-2 sweep reuses the histogram
#pragma unroll
    for (int u = 0; u < 4; ++u) row[u] = make_uint4(0u, 0u, 0u, 0u);
  unsigned tot = 0;
#pragma unroll
  for (int j = 0; j < 16; ++j) tot += c[j];
  unsigned incl = tot;  // slots in this lane's bins and above
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned v = __shfl_down_sync(0xffffffffu, incl, o);
    if (lane + o < 32) incl += v;
  }
  const unsigned need = static_cast<unsigned>(top_k - s.above);
  const unsigned above_lane = incl - tot;
  const bool mine = above_lane < need && need <= incl;
  int digit = 0;
  unsigned above = 0, cnt = 0;
  if (mine) {
    above = above_lane;
    int b = 15;
#pragma unroll 1
    for (; b > 0 && above + c[b] < need; --b) above += c[b];
    digit = lane * 16 + b;
    cnt = c[b];
  }
  const unsigned who = __ballot_sync(0xffffffffu, mine);
  const unsigned total = __shfl_sync(0xffffffffu, incl, 0);
  if (who) {
    const int src = __ffs(who) - 1;
    digit = __shfl_sync(0xffffffffu, digit, src);
    above = __shfl_sync(0xffffffffu, above, src);
    cnt = __shfl_sync(0xffffffffu, cnt, src);
  }
  if (lane != 0) return;
  const int64_t band = static_cast<int64_t>(s.above) + above + cnt;
  if (!who) {
    // fewer live slots than k (a device-side slot count below k): every slot is selected
    s.cut = 0u;
    s.mode = (LEVEL == 0 && total <= static_cast<unsigned>(kWideCap)) ? 0 : 2;
  } else if (LEVEL == 0) {
    if (band <= kWideCap) {
      s.cut = static_cast<unsigned>(digit) << kShift1;
      s.mode = 0;
    } else {
      s.d1 = digit;
      s.above = static_cast<int>(above);
      s.mode = 1;
    }
  } else {
    s.cut = (static_cast<unsigned>(s.d1) << kShift1) | (static_cast<unsigned>(digit) << kShift2);
    s.mode = band <= kWideCap ? 0 : 2;
  }
  state[lq] = s;
}

constexpr int S_THREADS = 256;

struct SelSmem {
  unsigned long long key[kWideCap];  // (~u << 32 | slot) ascending = the total order; later (slot << 32 | rank)
  float w[kWideMaxK];                // exp(s_j - s_0), rank order
  float qs[128];
  float out[512];
  unsigned hist[256];
  unsigned wcnt[S_THREADS / 32];
  unsigned prefix, need, n, ties;
  float sum;
};

__device__ __forceinline__ unsigned long long rank_key(float s, int slot) {
  return (static_cast<unsigned long long>(~score_key(s)) << 32) | static_cast<unsigned>(slot);
}
__device__ __forceinline__ float key_score(unsigned long long k) {
  return ordered_float(static_cast<int>(~static_cast<unsigned>(k >> 32) ^ 0x80000000u));
}

// Ascending bitonic sort of p (a power of two) keys by the whole block.
__device__ void block_sort(unsigned long long* k, int p) {
  for (int size = 2; size <= p; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < p / 2; i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
        const unsigned long long x = k[lo], y = k[hi];
        if ((x > y) == ((lo & size) == 0)) {
          k[lo] = y;
          k[hi] = x;
        }
      }
    }
  __syncthreads();
}

__device__ __forceinline__ int pow2_at_least(int n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

// Exact top-min(k, live) of one query into sm.key (unsorted): radix select over u, 8 bits per pass, every live slot
// re-scored in each pass, then the slots above the k-th key and the lowest-slot ties at it.  Returns the count.
__device__ int exact_topk(const MemreadArgs& a, int obj, int top_k, int64_t live, SelSmem& sm) {
  const int tid = threadIdx.x;
  const float* keys = a.bank_k + static_cast<int64_t>(obj) * a.slots_cap * 128;
  const int kk = static_cast<int>(top_k < live ? top_k : live);
  if (kk == 0) return 0;
  if (tid == 0) {
    sm.prefix = 0u;
    sm.need = static_cast<unsigned>(kk);
    sm.n = 0u;
    sm.ties = 0u;
  }
  unsigned mask = 0u;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += S_THREADS) sm.hist[i] = 0u;
    __syncthreads();
    const unsigned prefix = sm.prefix;
    for (int64_t s = tid; s < live; s += S_THREADS) {
      const unsigned u = score_key(exact_score(keys + s * 128, sm.qs));
      if ((u & mask) == prefix) atomicAdd(&sm.hist[(u >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      unsigned above = 0u, need = sm.need;
      int d = 255;
      for (; d > 0 && above + sm.hist[d] < need; --d) above += sm.hist[d];
      sm.need = need - above;
      sm.prefix = prefix | (static_cast<unsigned>(d) << shift);
    }
    mask |= 255u << shift;
    __syncthreads();
  }
  // sm.prefix is the k-th largest key T; sm.need of the slots with u == T belong to the top k (the lowest slots)
  const unsigned T = sm.prefix, need = sm.need;
  const int warp = tid >> 5, lane = tid & 31;
  for (int64_t s0 = 0; s0 < live; s0 += S_THREADS) {
    const int64_t s = s0 + tid;
    float sc = 0.f;
    unsigned u = 0u;
    if (s < live) {
      sc = exact_score(keys + s * 128, sm.qs);
      u = score_key(sc);
    }
    const bool tie = s < live && u == T;
    const unsigned bal = __ballot_sync(0xffffffffu, tie);
    if (lane == 0) sm.wcnt[warp] = __popc(bal);
    __syncthreads();
    unsigned before = sm.ties + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < warp; ++w) before += sm.wcnt[w];
    if ((s < live && u > T) || (tie && before < need)) sm.key[atomicAdd(&sm.n, 1u)] = rank_key(sc, static_cast<int>(s));
    __syncthreads();
    if (tid == 0)
      for (int w = 0; w < S_THREADS / 32; ++w) sm.ties += sm.wcnt[w];
    __syncthreads();
  }
  return static_cast<int>(sm.n);
}

__global__ void __launch_bounds__(S_THREADS)
memread_wide_select_kernel(const MemreadArgs a, const int top_k, const WideState* __restrict__ state,
                           const int2* __restrict__ cand, const int* __restrict__ cand_cnt, int* __restrict__ topk_idx,
                           float* __restrict__ topk_val) {
  mivos::pdl_prologue();
  extern __shared__ __align__(16) uint8_t sel_raw[];
  SelSmem& sm = *reinterpret_cast<SelSmem*>(sel_raw);
  const int tid = threadIdx.x;
  const int64_t lq = blockIdx.x;
  const int hw = a.hw;
  const int obj = static_cast<int>(lq / hw), q = static_cast<int>(lq - static_cast<int64_t>(obj) * hw);
  const int grp = object_group(a, obj);  // -1: in no group, reads set 0 over no slot
  const int qset = grp < 0 ? 0 : grp;
  const int64_t live = grp < 0 ? 0 : live_slots(a.dyn_slots, a.slots, a.slots_cap, grp, a.dyn_set_stride);

  int n;
  if (state[lq].mode != 2) {
    const int c = cand_cnt[lq];
    n = c < kWideCap ? c : kWideCap;  // the threshold stage sized every region: c <= kWideCap
    for (int i = tid; i < n; i += S_THREADS) {
      const int2 e = cand[lq * kWideCap + i];
      sm.key[i] = rank_key(__int_as_float(e.x), e.y);
    }
  } else {
    if (tid < 128) sm.qs[tid] = a.qk[(static_cast<int64_t>(qset) * hw + q) * 128 + tid] / kSqrtCK;
    __syncthreads();
    n = exact_topk(a, obj, top_k, live, sm);
  }
  const int p = pow2_at_least(n);
  for (int i = n + tid; i < p; i += S_THREADS) sm.key[i] = ~0ull;
  block_sort(sm.key, p);

  // ---- softmax over the first kk: exp(s - s_0) / sum (prop_net.py:55-58), the sum sequential in rank order
  const int kk = top_k < n ? top_k : n;
  const float s0 = kk > 0 ? key_score(sm.key[0]) : 0.f;
  for (int j = tid; j < kk; j += S_THREADS) sm.w[j] = expf(key_score(sm.key[j]) - s0);
  for (int t = tid; t < top_k; t += S_THREADS) {
    if (topk_idx) topk_idx[lq * top_k + t] = t < kk ? static_cast<int>(sm.key[t] & 0xffffffffu) : -1;
    if (topk_val) topk_val[lq * top_k + t] = t < kk ? key_score(sm.key[t]) : 0.f;
  }
  __syncthreads();
  if (tid == 0) {
    float sum = 0.f;
    for (int j = 0; j < kk; ++j) sum += sm.w[j];
    sm.sum = sum;
  }
  // ---- ascending slot order of the read-out
  const int p2 = pow2_at_least(kk);
  for (int j = tid; j < p2; j += S_THREADS)
    sm.key[j] = j < kk ? ((sm.key[j] & 0xffffffffull) << 32) | static_cast<unsigned>(j) : ~0ull;
  block_sort(sm.key, p2);
  const float sum = sm.sum;

  // ---- read-out: thread = channels 2 * tid, 2 * tid + 1; per channel the rows accumulate in ascending slot order
  const float2* vals = reinterpret_cast<const float2*>(a.bank_v + static_cast<int64_t>(obj) * a.slots_cap * 512);
  float2 acc = make_float2(0.f, 0.f);
  for (int j0 = 0; j0 < kk; j0 += 4) {
    float2 v[4];
    float w[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int jj = j0 + r < kk ? j0 + r : kk - 1;
      const unsigned long long e = sm.key[jj];
      w[r] = sm.w[static_cast<int>(e & 0xffffffffu)] / sum;
      v[r] = vals[static_cast<int64_t>(e >> 32) * 256 + tid];
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      if (j0 + r < kk) {
        acc.x = fmaf(w[r], v[r].x, acc.x);
        acc.y = fmaf(w[r], v[r].y, acc.y);
      }
    }
  }
  reinterpret_cast<float2*>(sm.out)[tid] = acc;
  __syncthreads();
  if (tid < 32) {
    float4 o[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) o[u] = reinterpret_cast<const float4*>(sm.out)[tid + 32 * u];
    store_read_row(a, obj, q, tid, o);
  }
}

// Workspace: level histograms [K*hw][512] u32 | emission counts [K*hw] | state [K*hw] | regions [K*hw][kWideCap]
// int2.  It depends on (objects, hw) alone.
struct WidePlan {
  int qtiles, splits;
  int64_t off_cnt, off_state, off_cand, bytes;
};

WidePlan wide_plan(int k_objects, int hw) {
  WidePlan pl;
  const int64_t nq = static_cast<int64_t>(k_objects) * hw;
  pl.qtiles = ceil_div(hw, WQ);
  // The sweep runs one CTA per SM: the fewest splits that fill the GPU and keep >= 90 % of the last wave busy (or the
  // best-filled count up to 64).  The memory axis is dealt to the splits tile by tile at run time.
  const int64_t sms = num_sms(), base = static_cast<int64_t>(pl.qtiles) * k_objects;
  pl.splits = 1;
  double best = 0.0;
  for (int s = 1; s <= 64; ++s) {
    const int64_t total = base * s;
    const double fill = static_cast<double>(total) / static_cast<double>(ceil_div64(total, sms) * sms);
    if (total >= sms && fill >= 0.9) {
      pl.splits = s;
      break;
    }
    if (fill > best + 1e-9) {
      best = fill;
      pl.splits = s;
    }
  }
  pl.off_cnt = nq * kBins * 4;
  pl.off_state = pl.off_cnt + ((nq * 4 + 255) & ~255ll);
  pl.off_cand = pl.off_state + ((nq * 16 + 255) & ~255ll);
  pl.bytes = pl.off_cand + nq * kWideCap * 8;
  return pl;
}

}  // namespace
}  // namespace mivos

using namespace mivos;

extern "C" MIVOS_API int64_t mivos_memory_read_wide_workspace(int k_objects, int64_t slots_cap, int hw, int top_k) {
  if (k_objects < 1 || k_objects > kMaxObjects || slots_cap < 1 || slots_cap >= (1ll << 31) - 65536 || hw < 1 ||
      top_k < 1 || top_k > kWideMaxK)
    return -1;
  return wide_plan(k_objects, hw).bytes;
}

namespace {

int memory_read_wide_run(const MemreadArgs& a, int top_k, int32_t* topk_idx, float* topk_val, void* workspace,
                         int64_t workspace_bytes, cudaStream_t stream) {
  MIVOS_REQUIRE(top_k >= 1 && top_k <= kWideMaxK, "memory_read_wide: top_k %d outside [1,%d]", top_k, kWideMaxK);
  MIVOS_REQUIRE(a.slots >= top_k && a.slots <= a.slots_cap && a.slots_cap < (1ll << 31) - 65536,
                "memory_read_wide: bad slot count %lld (cap %lld, k %d)", (long long)a.slots, (long long)a.slots_cap, top_k);
  MIVOS_REQUIRE(workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0,
                "memory_read_wide: workspace null or not 256-byte aligned");
  const WidePlan pl = wide_plan(a.k_objects, a.hw);
  MIVOS_REQUIRE(workspace_bytes >= pl.bytes, "memory_read_wide: workspace %lld < %lld bytes", (long long)workspace_bytes,
                (long long)pl.bytes);

  constexpr int hist_smem = static_cast<int>(sizeof(SweepSmem));
  constexpr int emit_smem = static_cast<int>(offsetof(SweepSmem, hist));
  constexpr int sel_smem = static_cast<int>(sizeof(SelSmem));
  static bool configured = false;
  if (!configured) {
    MIVOS_CUDA_OK(cudaFuncSetAttribute(memread_wide_sweep_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, hist_smem));
    MIVOS_CUDA_OK(cudaFuncSetAttribute(memread_wide_sweep_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, hist_smem));
    MIVOS_CUDA_OK(cudaFuncSetAttribute(memread_wide_sweep_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, emit_smem));
    MIVOS_CUDA_OK(cudaFuncSetAttribute(memread_wide_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sel_smem));
    configured = true;
  }
  uint8_t* w = static_cast<uint8_t*>(workspace);
  unsigned* hist = reinterpret_cast<unsigned*>(w);
  int* cnt = reinterpret_cast<int*>(w + pl.off_cnt);
  WideState* state = reinterpret_cast<WideState*>(w + pl.off_state);
  int2* cand = reinterpret_cast<int2*>(w + pl.off_cand);
  const int64_t nq = static_cast<int64_t>(a.k_objects) * a.hw;

  // histogram and emission counts start at zero (adjacent: one memset); the level-1 threshold clears each row it reads
  MIVOS_CUDA_OK(cudaMemsetAsync(w, 0, static_cast<size_t>(pl.off_state), stream));
  const dim3 grid(pl.qtiles, pl.splits, a.k_objects);
  const int tblocks = static_cast<int>(ceil_div64(nq, 8));
  launch_pdl(memread_wide_sweep_kernel<0>, grid, W_THREADS, hist_smem, stream, a, pl.splits,
             static_cast<const WideState*>(state), hist, cand, cnt);
  launch_pdl(memread_wide_threshold_kernel<0>, tblocks, 256, 0, stream, nq, top_k, state, hist);
  launch_pdl(memread_wide_sweep_kernel<1>, grid, W_THREADS, hist_smem, stream, a, pl.splits,
             static_cast<const WideState*>(state), hist, cand, cnt);
  launch_pdl(memread_wide_threshold_kernel<1>, tblocks, 256, 0, stream, nq, top_k, state, hist);
  launch_pdl(memread_wide_sweep_kernel<2>, grid, W_THREADS, emit_smem, stream, a, pl.splits,
             static_cast<const WideState*>(state), hist, cand, cnt);
  launch_pdl(memread_wide_select_kernel, static_cast<unsigned>(nq), S_THREADS, sel_smem, stream, a, top_k,
             static_cast<const WideState*>(state), static_cast<const int2*>(cand), static_cast<const int*>(cnt),
             topk_idx, topk_val);
  g_launches.fetch_add(6, std::memory_order_relaxed);
  MIVOS_CUDA_OK(cudaGetLastError());
  return MIVOS_OK;
}

}  // namespace

extern "C" MIVOS_API int mivos_memory_read_wide(const float* bank_k, const float* bank_v, int64_t slots_cap,
                                                int k_objects, int64_t slots, const float* qk, int hw, int q_div,
                                                int top_k, void* out, int out_cstride, int out_coff, int out_halo_h,
                                                int out_halo_w, int32_t* topk_idx, float* topk_val, void* workspace,
                                                int64_t workspace_bytes, const int32_t* dyn_slots, int out_f16,
                                                mivos_stream_t stream_) {
  const MemreadArgs a{bank_k, bank_v, slots_cap, k_objects, slots, dyn_slots, qk, hw, q_div,
                      out, out_cstride, out_coff, out_halo_h, out_halo_w, out_f16, 0};
  const int rc = memread_check_args(a, "memory_read_wide");
  if (rc != MIVOS_OK) return rc;
  return memory_read_wide_run(a, top_k, topk_idx, topk_val, workspace, workspace_bytes,
                              reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" MIVOS_API int mivos_memory_read_wide_sets(const float* bank_k, const float* bank_v, int64_t slots_cap,
                                                     int k_objects, int64_t slots, const float* qk, int hw, int sets,
                                                     int top_k, void* out, int out_cstride, int out_coff, int out_halo_h,
                                                     int out_halo_w, int32_t* topk_idx, float* topk_val, void* workspace,
                                                     int64_t workspace_bytes, const int32_t* dyn_slots, int out_f16,
                                                     mivos_stream_t stream_) {
  MemreadArgs a{bank_k, bank_v, slots_cap, k_objects, slots, dyn_slots, qk, hw, 0,
                out, out_cstride, out_coff, out_halo_h, out_halo_w, out_f16, 0};
  int rc = memread_sets_args(a, sets, "memory_read_wide_sets");
  if (rc == MIVOS_OK) rc = memread_check_args(a, "memory_read_wide_sets");
  if (rc != MIVOS_OK) return rc;
  return memory_read_wide_run(a, top_k, topk_idx, topk_val, workspace, workspace_bytes,
                              reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" MIVOS_API int mivos_memory_read_wide_groups(const float* bank_k, const float* bank_v, int64_t slots_cap,
                                                       int k_objects, int64_t slots, const float* qk, int hw, int groups,
                                                       const int32_t* first, int top_k, void* out, int out_cstride,
                                                       int out_coff, int out_halo_h, int out_halo_w, int32_t* topk_idx,
                                                       float* topk_val, void* workspace, int64_t workspace_bytes,
                                                       const int32_t* dyn_slots, int out_f16, mivos_stream_t stream_) {
  MemreadArgs a{bank_k, bank_v, slots_cap, k_objects, slots, dyn_slots, qk, hw, 0,
                out, out_cstride, out_coff, out_halo_h, out_halo_w, out_f16, 0};
  int rc = memread_check_args(a, "memory_read_wide_groups");
  if (rc == MIVOS_OK) rc = memread_groups_args(a, groups, first, "memory_read_wide_groups");
  if (rc != MIVOS_OK) return rc;
  return memory_read_wide_run(a, top_k, topk_idx, topk_val, workspace, workspace_bytes,
                              reinterpret_cast<cudaStream_t>(stream_));
}
