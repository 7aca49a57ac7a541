// Stage A2 of the memory read: candidate generation on the Hopper tensor cores.
//
// For one (object, 128-query tile, split of the memory axis) a CTA streams key tiles of 256 bank
// slots through TMA (128B swizzle) and computes the affinity tile
//     S[q, slot] = sum_c (qk[q,c]/sqrt(128)) * key[slot,c]
// with wgmma tf32 (two warpgroups of 64 queries each, N = 256 slots, K = 8 per instruction, 16
// instructions per tile) into register accumulators.  The query operand stays resident in shared
// memory (64 KB); keys flow through a 2-stage ring (2 x 32 KB) filled by one producer thread.
//
// Epilogue (in each warpgroup: two threads per query, one per column half of the slot tile): the
// accumulator fragment is transposed through a shared-memory tile, 64 columns per thread at a
// time, and each thread keeps
//   * NB "bucket maxima" in registers: NB values that are each a distinct score seen so far, so
//     the top_k-th largest of them (tau) is a LOWER bound of the top_k-th largest score of the
//     whole split.  (sorting them in place keeps the invariant; they are only ever max-updated.)
//     Two more bounds tighten it at every refresh: the PAIR bound (min over the two halves of their
//     ceil(k/2)-th bucket maximum: disjoint slots, so k scores >= it) and whatever any other CTA working
//     on the same query has published (one atomicMax word per (object, query)).
//   * a candidate list in global memory: every score >= tau - margin is appended (PTX: one compare,
//     one predicated 8-byte store, one predicated bump of the low address word).
// TF32 operand truncation makes S approximate; margin = 2*eps with the rigorous bound
//   eps = 1.05 * 2^-9 * ||q/sqrt(128)|| * max_slot ||key||      (Cauchy-Schwarz over channels)
// guarantees every member of the exact fp32 top-k is emitted.  Stage B re-scores the survivors in
// exact fp32 (memread.cu), so the final indices/weights do not depend on TF32 at all.
// The first WARM tiles only build tau; they are replayed (one extra MMA tile each) at the end
// with the final threshold (emission only — the replay does not touch the bucket maxima).  Lists
// are left as written: the selection stage filters them against the final shared threshold.
// A list that would overflow while streaming raises a per-query flag; flagged queries — and those
// the selection stage flags because their lists hold more in-band candidates than it can stage —
// are served by the exact CUDA-core path (memread_exact_kernel + selection pass B), so adversarial
// inputs (all-equal keys, huge-norm keys) stay correct.
//
// Roofline: tensor pipe.  Algorithmic flops 2*128*slots*hw per object.
#include "pdl.cuh"
#include "memread.h"
#include "sm90.cuh"

#include <atomic>
#include <cstdlib>

namespace mivos {
extern std::atomic<int64_t> g_launches;
namespace {

constexpr int TQ = 128;
constexpr int TS = 256;
constexpr int KB = 32;
constexpr int NKB = 4;
constexpr int STAGES = 2;
constexpr int QBLK_BYTES = TQ * KB * 4;       // 16 KB per k-block of the query tile
constexpr int Q_BYTES = QBLK_BYTES * NKB;     // 64 KB
constexpr int STAGE_BYTES = TS * KB * 4;      // 32 KB
constexpr int WARM = 2;
constexpr int TC_THREADS = 288;              // 2 MMA / epilogue warpgroups, TMA producer warp
constexpr int STREAM_CAP = kTcCandCap;        // per (object, query, split) while streaming
constexpr float kSqrtCK = 11.313708498984761f;
constexpr float kEpsFactor = kTcMarginFactor;

struct TcParams {
  int64_t slots_cap, slots;
  int hw, top_k, splits, nlists, tiles_per_split;
  int q_div;            // objects per query set (lock-step clips: K objects of a clip share its query); 0 = one set
  const int* dyn_slots;  // optional device scalar overriding `slots` (CUDA-graph replay)
  const float* qnorm;   // [hw]   ||q/sqrt(128)||
  const float* kmax2;   // [K]    max_slot ||key||^2 (as float)
  int2* cand;  // lists of {score bits, slot}
  int* cand_cnt;
  int* overflow;        // [K*hw]
  int* tau_g;           // [K*hw] order-preserving int encoding of the best threshold any CTA has found
  int* err;
  unsigned spin_ns;     // sleep between barrier polls of the TMA / MMA threads (0 = poll flat out)
};

// float <-> int with the same ordering (so atomicMax on the int is a max on the float)
__device__ __forceinline__ int float_ordered(float f) {
  const int b = __float_as_int(f);
  return b >= 0 ? b : b ^ 0x7fffffff;
}
__device__ __forceinline__ float ordered_float(int o) { return __int_as_float(o >= 0 ? o : o ^ 0x7fffffff); }

// ---- prep: scaled queries, their norms, and the max key norm per object --------------------
__global__ void memread_prep_kernel(const float* __restrict__ qk, int hw, int q_rows, int q_div, float* __restrict__ qs,
                                    float* __restrict__ qnorm, const float* __restrict__ bank_k,
                                    int64_t slots_cap, int64_t slots, int k_objects,
                                    unsigned int* __restrict__ kmax2_bits, int qblocks,
                                    const int* __restrict__ dyn_slots, int* __restrict__ tau_g) {
  mivos::pdl_prologue();
  if (dyn_slots) slots = *dyn_slots;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (static_cast<int>(blockIdx.x) < qblocks) {
    // one warp per query row r = set * hw + q
    const int r = blockIdx.x * 8 + warp;
    if (r < q_rows) {
      const float4 v = reinterpret_cast<const float4*>(qk + static_cast<int64_t>(r) * 128)[lane];
      float4 s;
      s.x = v.x / kSqrtCK; s.y = v.y / kSqrtCK; s.z = v.z / kSqrtCK; s.w = v.w / kSqrtCK;
      reinterpret_cast<float4*>(qs + static_cast<int64_t>(r) * 128)[lane] = s;
      float n2 = s.x * s.x + s.y * s.y + s.z * s.z + s.w * s.w;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, o);
      if (lane == 0) qnorm[r] = sqrtf(n2) * 1.0001f;  // round the bound up
      // shared thresholds of the objects that read this query set start at the lowest value
      const int set = r / hw, q = r - set * hw;
      const int o0 = q_div > 0 ? set * q_div : 0;
      int o1 = q_div > 0 ? o0 + q_div : k_objects;
      if (o1 > k_objects) o1 = k_objects;
      for (int o = o0 + lane; o < o1; o += 32) tau_g[static_cast<int64_t>(o) * hw + q] = float_ordered(-3.0e38f);
    }
    return;
  }
  // key norms: grid-stride over (object, slot), one warp per row, block-level max then atomic
  const int nb = gridDim.x - qblocks;
  const int b = blockIdx.x - qblocks;
  for (int obj = 0; obj < k_objects; ++obj) {
    float best = 0.f;
    for (int64_t s = static_cast<int64_t>(b) * 8 + warp; s < slots; s += static_cast<int64_t>(nb) * 8) {
      const float4 v = reinterpret_cast<const float4*>(bank_k + (static_cast<int64_t>(obj) * slots_cap + s) * 128)[lane];
      float n2 = v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, o);
      best = fmaxf(best, n2);
    }
    if (lane == 0) atomicMax(kmax2_bits + obj, __float_as_uint(best * 1.0001f));  // non-negative floats order as uints
  }
}

// ---- in-register bitonic sort, descending --------------------------------------------------
template <int N>
__device__ __forceinline__ void sort_desc(float (&x)[N]) {
#pragma unroll
  for (int size = 2; size <= N; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
#pragma unroll
      for (int i = 0; i < N; ++i) {
        const int j = i ^ stride;
        if (j > i) {
          const bool desc = ((i & size) == 0);
          const float a = x[i], b = x[j];
          const float hi = fmaxf(a, b), lo = fminf(a, b);
          x[i] = desc ? hi : lo;
          x[j] = desc ? lo : hi;
        }
      }
    }
  }
}

template <int NB>
__device__ __forceinline__ float kth_largest(float (&m)[NB], int k) {
  sort_desc<NB>(m);
  float t = m[NB - 1];
#pragma unroll
  for (int i = 0; i < NB; ++i)
    if (i == k - 1) t = m[i];
  return t;
}

// k-th and kh-th largest bucket maxima in one sort (kh <= k)
template <int NB>
__device__ __forceinline__ void kth_pair(float (&m)[NB], int k, int kh, float& t_k, float& t_kh) {
  sort_desc<NB>(m);
  t_k = m[NB - 1];
  t_kh = m[NB - 1];
#pragma unroll
  for (int i = 0; i < NB; ++i) {
    if (i == k - 1) t_k = m[i];
    if (i == kh - 1) t_kh = m[i];
  }
}

// In-place filter of a thread's own candidate list (global memory).  Loads are issued four
// entries ahead of the stores so the loop is not one dependent L2 round trip per entry; stores go
// to indices <= the entries already read, so batching is safe.
__device__ __forceinline__ int compact_list(int2* list, int cnt, float thr) {
  int n = 0;
  int j = 0;
  for (; j + 4 <= cnt; j += 4) {
    int2 e[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) e[u] = __ldcg(list + j + u);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (__int_as_float(e[u].x) >= thr) list[n++] = e[u];
    }
  }
  for (; j < cnt; ++j) {
    const int2 e = __ldcg(list + j);
    if (__int_as_float(e.x) >= thr) list[n++] = e;
  }
  return n;
}

// Append {score bits, slot} to the thread's list if the score passes.  Written in PTX so that it stays what it says:
// one compare, one predicated 8-byte store, one predicated 64-bit bump.  (The C++ form of the same statement was
// compiled into a 32-element prefix sum over materialised predicates with the addresses rebuilt per element:
// ~15 instructions per tested score; the epilogue is what bounds this kernel.)
// `lo` / `hi` are the halves of the append address: a list never straddles a 4 GB boundary (plan_lists), so only
// the low word moves.
__device__ __forceinline__ void emit_if_ge(int2*& lp, float v, float tau, int slot) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      ".reg .b32 l, h;\n"
      "setp.ge.f32 p, %1, %2;\n"
      "@p st.global.v2.b32 [%0], {%3, %4};\n"
      "mov.b64 {l, h}, %0;\n"
      "@p add.u32 l, l, 8;\n"
      "mov.b64 %0, {l, h};\n"
      "}\n"
      : "+l"(lp)
      : "f"(v), "f"(tau), "r"(__float_as_int(v)), "r"(slot)
      : "memory");
}

// Query rows of a warpgroup's 64 x 128 staging tile: columns [0, 64) of the chunk for half 0, [64, 128) for half 1;
// the pad makes the fragment stores (8-byte pieces of 4 rows per half-warp) conflict-free.
constexpr int STG_STRIDE = 136;
constexpr int STG_BYTES = 64 * STG_STRIDE * 4;

// Register budget: 168 per thread.  An SM's register file is split over its four scheduler partitions (16384
// each); 9 warps put 3 on one partition, so 16384 / (3 x 32) caps a thread at 168 — a larger cap compiles but the
// launch is refused.  The 128-float accumulator fragment, the NB bucket maxima and a 32-score chunk do not all fit
// there: ptxas spills 0.3-1.3 KB per thread (NB = 32 / 64), served from L1, inside the candidate loop.
template <int NB, bool EMIT_PTX>
__global__ void __launch_bounds__(TC_THREADS, 1)
memread_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                  const TcParams p) {
  mivos::pdl_prologue();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_k = smem + Q_BYTES;
  float* stg_all = reinterpret_cast<float*>(smem + Q_BYTES + STAGES * STAGE_BYTES);  // [2 warpgroups][64][STG_STRIDE]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Q_BYTES + STAGES * STAGE_BYTES + 2 * STG_BYTES);
  uint64_t* q_full = bars;
  uint64_t* full_bar = bars + 1;
  uint64_t* empty_bar = full_bar + STAGES;
  float* tau_x = reinterpret_cast<float*>(empty_bar + STAGES);  // [2][kTcHalves][128] thresholds exchanged between the halves

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * TQ;
  const int split = blockIdx.y;
  const int obj = blockIdx.z;
  const int qrow0 = (p.q_div > 0 ? obj / p.q_div : 0) * p.hw;  // first row of this object's query set
  const int64_t slots = p.dyn_slots ? static_cast<int64_t>(*p.dyn_slots) : p.slots;
  const int total_tiles = static_cast<int>((slots + TS - 1) / TS);
  // with a device-side slot count the grid (splits) is fixed by the host for the bank capacity and
  // the tile ranges are derived here; splits beyond the live bank publish empty lists and leave
  const int tps = p.dyn_slots ? (total_tiles + p.splits - 1) / p.splits : p.tiles_per_split;
  const int t_begin = split * tps;
  int t_end = t_begin + tps;
  if (t_end > total_tiles) t_end = total_tiles;
  const int nloc = t_end - t_begin;
  // MMA / epilogue warpgroups 0 and 1 (warps 0-7): queries [0, 64) and [64, 128) of the tile; in each, warps 0-1 own
  // the column half [0, 128) of every slot tile and warps 2-3 the half [128, 256), one query per thread.  Warp 8 is
  // the TMA producer (see the register budget above the kernel)
  const int wg = warp / 4;
  const int tw = threadIdx.x & 127;
  const int half = tw >> 6;
  const int qi = wg * 64 + (tw & 63);  // query of this thread within the tile
  if (nloc <= 0) {
    if (warp < 8) {
      const int qq = q0 + qi;
      if (qq < p.hw) p.cand_cnt[(static_cast<int64_t>(obj) * p.hw + qq) * p.nlists + split * kTcHalves + half] = 0;
    }
    return;
  }
  const int warm = nloc < WARM ? nloc : WARM;
  const int nseq = nloc + warm;

  if (threadIdx.x == 0) {
    sm90::prefetch_tmap(&tmQ);
    sm90::prefetch_tmap(&tmK);
    sm90::mbar_init(q_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      sm90::mbar_init(&full_bar[s], 1);
      sm90::mbar_init(&empty_bar[s], 8);  // one arrival per MMA warp
    }
    sm90::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      sm90::mbar_arrive_expect_tx(q_full, Q_BYTES);
      // (the last tile of a set may run into the next set's rows: those lanes are masked by `valid`)
      for (int kb = 0; kb < NKB; ++kb) sm90::tma_load_2d(smem_q + kb * QBLK_BYTES, &tmQ, q_full, kb * KB, qrow0 + q0);
      const int64_t row0 = static_cast<int64_t>(obj) * p.slots_cap;
      int it = 0;
      for (int i = 0; i < nseq; ++i) {
        const int tile = t_begin + (i < nloc ? i : i - nloc);
        const int32_t row = static_cast<int32_t>(row0 + static_cast<int64_t>(tile) * TS);
        for (int kb = 0; kb < NKB; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          if (p.spin_ns) sm90::mbar_wait_backoff(&empty_bar[s], ph ^ 1, p.err, 301, p.spin_ns);
          else sm90::mbar_wait(&empty_bar[s], ph ^ 1, p.err, 301);
          sm90::mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
          sm90::tma_load_2d(smem_k + s * STAGE_BYTES, &tmK, &full_bar[s], kb * KB, row);
        }
      }
    }
    return;
  }

  const uint32_t bar_id = 1 + wg;  // named barrier of this warpgroup
  float* const stg = stg_all + wg * 64 * STG_STRIDE;
  const int q = q0 + qi;
  const bool valid = q < p.hw;
  const int64_t lq = static_cast<int64_t>(obj) * p.hw + (valid ? q : 0);
  const float margin = valid ? kEpsFactor * p.qnorm[qrow0 + q] * sqrtf(p.kmax2[obj]) : 0.f;
  const int64_t list_id = lq * p.nlists + split * kTcHalves + half;
  int2* const list = p.cand + list_id * STREAM_CAP;
  int2* lp = list;  // append pointer (count = lp - list)
  float m[NB];
#pragma unroll
  for (int b = 0; b < NB; ++b) m[b] = -INFINITY;
  float tau_emit = -INFINITY;
  bool overflow = false;
  int retau_n = 0;
  float acc[TS / 2];  // wgmma fragment of the 64 x 256 score tile
  sm90::mbar_wait(&q_full[0], 0, p.err, 302);
  const uint32_t q_addr = sm90::smem_u32(smem_q) + wg * 64 * 128;
  // fragment coordinates of this thread: rows fr, fr + 8, columns 8j + fc, 8j + fc + 1
  const int fr = (tw >> 5) * 16 + ((tw & 31) >> 2);
  const int fc = 2 * (tw & 3);

  int it = 0;
  for (int i = 0; i < nseq; ++i) {
    int prev = -1;
    // (the first wgmma overwrites the fragment: zeroing it here tells the compiler that the previous tile's values
    // are dead, so they do not occupy registers across the threshold refresh)
#pragma unroll
    for (int j = 0; j < TS / 2; ++j) acc[j] = 0.f;
    for (int kb = 0; kb < NKB; ++kb, ++it) {
      const int s = it % STAGES;
      sm90::mbar_wait(&full_bar[s], (it / STAGES) & 1, p.err, 304);
      const uint64_t da = sm90::make_desc_sw128(q_addr + kb * QBLK_BYTES);
      const uint64_t db = sm90::make_desc_sw128(sm90::smem_u32(smem_k + s * STAGE_BYTES));
      sm90::wgmma_fence();
#pragma unroll
      for (int k = 0; k < KB / 8; ++k) sm90::wgmma<TS, false>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
      sm90::wgmma_commit();
      sm90::wgmma_wait<1>();  // the previous k-block's wgmmas are done: its stage may be refilled
      if (prev >= 0 && lane == 0) sm90::mbar_arrive(&empty_bar[prev]);
      prev = s;
    }
    sm90::wgmma_wait<0>();
    sm90::fence_acc(acc);
    if (lane == 0) sm90::mbar_arrive(&empty_bar[prev]);

    const int tile = t_begin + (i < nloc ? i : i - nloc);
    const int64_t slot0 = static_cast<int64_t>(tile) * TS;
    const int64_t rem = slots - slot0;
    const int ncols = rem < TS ? static_cast<int>(rem) : TS;
    const bool emit = (i >= warm) && valid && !overflow;
    // Two chunks: chunk c holds columns [64c, 64c + 64) of half 0 and [128 + 64c, ...) of half 1; the warpgroup parks
    // them in its staging tile and every thread reads back the 64 scores of its own query and half, 32 at a time.
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      sm90::named_sync(bar_id, 128);  // the previous chunk has been read
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int j = h * 16 + 8 * c + jj;
          float* dst = stg + fr * STG_STRIDE + h * 64 + 8 * jj + fc;
          *reinterpret_cast<float2*>(dst) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(dst + 8 * STG_STRIDE) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      sm90::named_sync(bar_id, 128);
#pragma unroll
      for (int sb = 0; sb < 2; ++sb) {
        float v[32];
        const float* src = stg + (tw & 63) * STG_STRIDE + half * 64 + sb * 32;
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const float4 t = *reinterpret_cast<const float4*>(src + j);
          v[j] = t.x; v[j + 1] = t.y; v[j + 2] = t.z; v[j + 3] = t.w;
        }
        const int col0 = half * (TS / kTcHalves) + c * 64 + sb * 32;  // tile column of v[0]
        if (col0 + 32 > ncols) {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (col0 + j >= ncols) v[j] = -INFINITY;  // stale rows past the live bank
        }
        // bucket maxima (bucket = column mod NB).  NOT on the replayed warm tiles: m[] is sorted in place between
        // tiles, so re-presenting an element already witnessed could store it in a second position and break the
        // "NB distinct scores" invariant that makes tau a lower bound.
        if (i < nloc) {
          const int off = (NB == 64 && sb) ? 32 : 0;  // a constant once unrolled
#pragma unroll
          for (int j = 0; j < 32; ++j) m[(off + j) % NB] = fmaxf(m[(off + j) % NB], v[j]);
        }
        if (emit) {
          const int idx0 = static_cast<int>(slot0) + col0;
          if constexpr (EMIT_PTX) {
#pragma unroll
            for (int j = 0; j < 32; ++j) emit_if_ge(lp, v[j], tau_emit, idx0 + j);
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const bool pass = v[j] >= tau_emit;
              if (pass) *lp = make_int2(__float_as_int(v[j]), idx0 + j);
              lp += pass ? 1 : 0;
            }
          }
        }
      }
    }

    // threshold schedule: end of warm-up, then every 4th tile, and before the replay
    const bool retau = (i + 1 == warm) || (i + 1 > warm && ((i + 1 - warm) & 3) == 0) || (i + 1 == nloc);
    // clamp above -inf: masked (stale) columns carry -inf and must never pass `v >= tau_emit`
    if (retau) {
      // Any subset's k-th largest score is a lower bound of the global k-th largest, so the best
      // bound found by ANY CTA working on this query (other splits, the other column half) is as
      // valid as our own: share it through one atomicMax per refresh.  This is what keeps the
      // lists short: without it every list keeps what beats ITS OWN k-th score.  Which bound is
      // visible when is a matter of timing, so list lengths vary from run to run; the selected
      // top-k does not.
      // A second, tighter bound from the PAIR of column halves: they saw disjoint slots, so if this half holds
      // ceil(k/2) distinct scores >= a and the other ceil(k/2) distinct scores >= b, the two together hold k
      // scores >= min(a, b).
      float t, t_half;
      kth_pair<NB>(m, p.top_k, (p.top_k + 1) >> 1, t, t_half);
      {
        float* tx = tau_x + (retau_n & 1) * (kTcHalves * 128);  // two buffers: one barrier per exchange
        ++retau_n;
        tx[half * 128 + qi] = t_half;
        sm90::named_sync(bar_id, 128);  // both halves of a query are in this warpgroup
        float pair = t_half;
#pragma unroll
        for (int hh = 0; hh < kTcHalves; ++hh) pair = fminf(pair, tx[hh * 128 + qi]);
        t = fmaxf(t, pair);
      }
      if (valid) {
        const int enc = float_ordered(fmaxf(t, -3.0e38f));
        const int prev_t = atomicMax(p.tau_g + lq, enc);
        t = ordered_float(prev_t > enc ? prev_t : enc);
      }
      tau_emit = fmaxf(t - margin, -3.0e38f);
    }
    // keep room for this thread's share of a full tile of appends
    if ((lp - list) > STREAM_CAP - TS / kTcHalves && !overflow) {
      const int kept = compact_list(list, static_cast<int>(lp - list), tau_emit);
      lp = list + kept;
      if (kept > STREAM_CAP - TS / kTcHalves) overflow = true;
    }
  }
  // Final threshold: both column halves saw disjoint parts of the same split, each tau is a
  // lower bound of the split's k-th largest score, hence so is their maximum.
  // (the last refresh of the loop ran at i + 1 == nloc, before the replayed tiles, which do not touch m[]:
  // tau_g already holds this CTA's final bounds, the pair bound included)
  float tau_fin = kth_largest<NB>(m, p.top_k);
  if (valid) tau_fin = fmaxf(tau_fin, ordered_float(__ldcg(p.tau_g + lq)));
  if (valid) {
    // Lists are left as they are: the selection stage filters them against the final shared threshold anyway, and
    // it is the selection stage that sends a query whose lists carry more in-band candidates than it can hold to
    // the exact CUDA-core path (memread.cu, pass A).  Only a list that overflowed while streaming flags here.
    p.cand_cnt[list_id] = overflow ? 0 : static_cast<int>(lp - list);
    if (overflow) atomicExch(p.overflow + lq, 1);
  }
}

constexpr int TC_SMEM = Q_BYTES + STAGES * STAGE_BYTES + 2 * STG_BYTES + (1 + 2 * STAGES) * 8 + 2 * 128 * kTcHalves * 4 + 1024;

}  // namespace

bool memread_tc_available() { return true; }

int memread_tc_run(const float* bank_k, const float* bank_v, int64_t slots_cap, int k_objects,
                   int64_t slots, const float* qk, int hw, int q_div, int top_k, void* out, int out_cstride,
                   int out_coff, int halo_h, int halo_w, int out_f16, int32_t* topk_idx, float* topk_val,
                   void* workspace, const int* dyn_slots, cudaStream_t stream) {
  MIVOS_REQUIRE(static_cast<int64_t>(k_objects) * slots_cap < (1ll << 31) - 4096,
                "memory_read(tensor cores): bank rows exceed int32 TMA coordinates");
  const MemreadPlan tc = memread_plan(k_objects, slots, hw, top_k, MIVOS_MEMREAD_TCGEN05);
  const MemreadPlan ex = memread_plan(k_objects, slots, hw, top_k, MIVOS_MEMREAD_EXACT_SIMT);
  uint8_t* w = static_cast<uint8_t*>(workspace);
  uint8_t* w_tc = w;
  uint8_t* w_ex = w + tc.bytes;
  const int q_sets = q_div > 0 ? ceil_div(k_objects, q_div) : 1;
  const int q_rows = q_sets * hw;
  MIVOS_REQUIRE(k_objects <= kMaxObjects, "memory_read: more than %d objects in one call", kMaxObjects);
  // tail of the workspace (sized for k_objects query sets): flags | key-norm maxima | scaled queries | norms | tau
  const int64_t nq = static_cast<int64_t>(k_objects) * hw, nq64 = (nq + 63) & ~63ll;  // arrays padded to 256 bytes
  int* flags = reinterpret_cast<int*>(w + tc.bytes + ex.bytes);
  unsigned int* kmax2 = reinterpret_cast<unsigned int*>(flags + nq64);
  float* qs = reinterpret_cast<float*>(kmax2 + kMaxObjects);  // 16-byte aligned: TMA source, float4 stores
  float* qnorm = qs + nq * 128;
  int* tau_g = reinterpret_cast<int*>(qnorm + nq64);

  // overflow flags (written here and by the first selection pass, read by the exact fallback and the second selection
  // pass) and the key-norm accumulator start at zero: ONE memset over the two adjacent arrays
  MIVOS_CUDA_OK(cudaMemsetAsync(flags, 0, static_cast<size_t>(nq64 + kMaxObjects) * 4, stream));

  const int qblocks = ceil_div(q_rows, 8);
  const int kblocks = 296;
  launch_pdl(memread_prep_kernel, qblocks + kblocks, 256, 0, stream, qk, hw, q_rows, q_div, qs, qnorm, bank_k, slots_cap, slots,
                                                             k_objects, kmax2, qblocks, dyn_slots, tau_g);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  MIVOS_CUDA_OK(cudaGetLastError());

  CUtensorMap tmQ, tmK;
  int rc = encode_tmap_2d(&tmQ, qs, static_cast<uint64_t>(q_rows), 128, 128, KB, TQ);
  if (rc != MIVOS_OK) return rc;
  rc = encode_tmap_2d(&tmK, bank_k, static_cast<uint64_t>(k_objects) * slots_cap, 128, 128, KB, TS);
  if (rc != MIVOS_OK) return rc;

  TcParams p;
  p.slots_cap = slots_cap;
  p.slots = slots;
  p.dyn_slots = dyn_slots;
  p.hw = hw;
  p.q_div = q_div;
  p.top_k = top_k;
  p.splits = tc.splits;
  p.nlists = tc.nlists;
  p.tiles_per_split = tc.tiles_per_split;
  p.qnorm = qnorm;
  p.kmax2 = reinterpret_cast<const float*>(kmax2);
  p.cand = reinterpret_cast<int2*>(plan_lists(w_tc, tc));
  p.cand_cnt = reinterpret_cast<int*>(w_tc + tc.off_cnt);
  p.overflow = flags;
  p.tau_g = tau_g;
  p.err = device_error_flag();

  // MIVOS_MEMREAD_EMIT=c selects the compiler's emission loop, MIVOS_MEMREAD_BACKOFF_NS the producer's sleep
  // between barrier polls (0 = poll flat out)
  static const bool emit_ptx = [] { const char* e = getenv("MIVOS_MEMREAD_EMIT"); return !(e && e[0] == 'c'); }();
  static const unsigned spin_ns = [] { const char* e = getenv("MIVOS_MEMREAD_BACKOFF_NS"); return e ? static_cast<unsigned>(atoi(e)) : 100u; }();
  p.spin_ns = spin_ns;

  static bool configured = false;
  if (!configured) {
    MIVOS_CUDA_OK(cudaFuncSetAttribute(memread_tc_kernel<32, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
    MIVOS_CUDA_OK(cudaFuncSetAttribute(memread_tc_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
    MIVOS_CUDA_OK(cudaFuncSetAttribute(memread_tc_kernel<32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
    MIVOS_CUDA_OK(cudaFuncSetAttribute(memread_tc_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
    configured = true;
  }
  dim3 grid(tc.qtiles, tc.splits, k_objects);
  if (top_k <= 32) {
    if (emit_ptx) launch_pdl(memread_tc_kernel<32, true>, grid, TC_THREADS, TC_SMEM, stream, tmQ, tmK, p);
    else launch_pdl(memread_tc_kernel<32, false>, grid, TC_THREADS, TC_SMEM, stream, tmQ, tmK, p);
  } else {
    if (emit_ptx) launch_pdl(memread_tc_kernel<64, true>, grid, TC_THREADS, TC_SMEM, stream, tmQ, tmK, p);
    else launch_pdl(memread_tc_kernel<64, false>, grid, TC_THREADS, TC_SMEM, stream, tmQ, tmK, p);
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  MIVOS_CUDA_OK(cudaGetLastError());

  // selection pass A: every query the candidate pass did not flag, from the tensor-core lists; a query whose lists carry
  // more in-band candidates than the stage can hold is flagged there instead of being selected
  rc = launch_select(bank_k, bank_v, slots_cap, k_objects, qk, hw, q_div, top_k, tc, w_tc, nullptr, nullptr, flags, 0, qnorm,
                     reinterpret_cast<const float*>(kmax2), tau_g, out, out_cstride, out_coff, halo_h, halo_w, out_f16, topk_idx,
                     topk_val, stream);
  if (rc != MIVOS_OK) return rc;
  // exact fallback for flagged queries only (CTAs without a flagged query exit immediately) ...
  rc = launch_exact_candidates(bank_k, slots_cap, k_objects, slots, qk, hw, q_div, top_k, ex, w_ex, flags, dyn_slots, stream);
  if (rc != MIVOS_OK) return rc;
  // ... and selection pass B: the flagged queries, from the exact lists (warps of the others leave at once)
  return launch_select(bank_k, bank_v, slots_cap, k_objects, qk, hw, q_div, top_k, ex, w_ex, nullptr, nullptr, flags, 1, nullptr,
                       nullptr, nullptr, out, out_cstride, out_coff, halo_h, halo_w, out_f16, topk_idx, topk_val, stream);
}

}  // namespace mivos
