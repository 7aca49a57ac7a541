// Fusion attention map: PropagationNetwork.get_attention + AttentionMemory.forward of the
// reference (model/propagation/prop_net.py:115-129, 187-200).
//   W[i, j] = softmax_i( mk[:, i] . qk[:, j] / sqrt(128) )            (T = 1, no top-k)
//   pos_map[j] = sum_i area16(pos)[i] * W[i, j]   (same for neg);  bilinear x16 to (H, W).
// W (hw x hw) is never written to memory: one CTA owns 8 query columns, keeps their logits in
// shared memory and reduces them against the two pooled difference masks.
// 0.68 GFLOP at 480p: a CUDA-core kernel, only reached on the fusion path (cfg-4).
#include "host_util.h"
#include "pdl.cuh"

#include <atomic>
#include <mutex>

namespace mivos {
extern std::atomic<int64_t> g_launches;
namespace {

constexpr float kSqrtCK = 11.313708498984761f;
constexpr int QB = 8;  // queries per CTA
constexpr int ATT_THREADS = 256;

// adaptive average pool 16x16 -> pooled[2][hw] (F.interpolate(mode='area'), prop_net.py:194-195)
__global__ void area_pool16_kernel(const float* __restrict__ pos, const float* __restrict__ neg,
                                   int h16, int w16, float* __restrict__ pooled) {
  mivos::pdl_prologue();
  const int hw = h16 * w16;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * hw) return;
  const float* src = (i < hw) ? pos : neg;
  const int cell = (i < hw) ? i : i - hw;
  const int cy = cell / w16, cx = cell - cy * w16;
  const int W = w16 * 16;
  float s = 0.f;
  for (int y = 0; y < 16; ++y)
    for (int x = 0; x < 16; ++x) s += src[static_cast<int64_t>(cy * 16 + y) * W + cx * 16 + x];
  pooled[i] = s / 256.f;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(ATT_THREADS)
attention_kernel(const float* __restrict__ mk, const float* __restrict__ qk, int hw,
                 const float* __restrict__ pooled, float* __restrict__ maps, float* __restrict__ w_out) {
  mivos::pdl_prologue();
  extern __shared__ __align__(16) float sm[];
  float* qs = sm;                // [QB][128]
  float* S = sm + QB * 128;      // [QB][hw]
  __shared__ float m_s[QB], den_s[QB];
  const int tid = threadIdx.x;
  const int j0 = blockIdx.x * QB;
  for (int i = tid; i < QB * 128; i += ATT_THREADS) {
    const int q = i >> 7, c = i & 127;
    qs[i] = (j0 + q < hw) ? qk[static_cast<int64_t>(j0 + q) * 128 + c] / kSqrtCK : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < hw; i += ATT_THREADS) {
    float acc[QB];
#pragma unroll
    for (int q = 0; q < QB; ++q) acc[q] = 0.f;
    const float4* krow = reinterpret_cast<const float4*>(mk + static_cast<int64_t>(i) * 128);
#pragma unroll 4
    for (int c4 = 0; c4 < 32; ++c4) {
      const float4 kv = krow[c4];
#pragma unroll
      for (int q = 0; q < QB; ++q) {
        const float4 qv = *reinterpret_cast<const float4*>(qs + q * 128 + c4 * 4);
        acc[q] = fmaf(kv.x, qv.x, acc[q]);
        acc[q] = fmaf(kv.y, qv.y, acc[q]);
        acc[q] = fmaf(kv.z, qv.z, acc[q]);
        acc[q] = fmaf(kv.w, qv.w, acc[q]);
      }
    }
#pragma unroll
    for (int q = 0; q < QB; ++q) S[q * hw + i] = acc[q];
  }
  __syncthreads();
  // one warp per query column: softmax over the memory axis, reduced against pooled pos / neg
  const int warp = tid >> 5, lane = tid & 31;
  if (warp < QB && j0 + warp < hw) {
    const float* s = S + warp * hw;
    float m = -INFINITY;
    for (int i = lane; i < hw; i += 32) m = fmaxf(m, s[i]);
    m = warp_max(m);
    float den = 0.f, pp = 0.f, nn = 0.f;
    for (int i = lane; i < hw; i += 32) {
      const float e = expf(s[i] - m);
      den += e;
      pp = fmaf(e, pooled[i], pp);
      nn = fmaf(e, pooled[hw + i], nn);
    }
    den = warp_sum(den);
    pp = warp_sum(pp);
    nn = warp_sum(nn);
    if (lane == 0) {
      maps[j0 + warp] = pp / den;
      maps[hw + j0 + warp] = nn / den;
      m_s[warp] = m;
      den_s[warp] = den;
    }
  }
  if (w_out) {
    // get_W (prop_net.py:183): the affinity itself, [hw (memory), hw (query)] row-major; a thread
    // writes the QB consecutive query columns of one memory row
    __syncthreads();
    const int nq = hw - j0 < QB ? hw - j0 : QB;
    for (int i = tid; i < hw; i += ATT_THREADS)
      for (int q = 0; q < nq; ++q)
        w_out[static_cast<int64_t>(i) * hw + j0 + q] = expf(S[q * hw + i] - m_s[q]) / den_s[q];
  }
}

// bilinear [2][h16][w16] -> [2][H][W], align_corners=False (prop_net.py:198)
__global__ void upsample16_kernel(const float* __restrict__ maps, int h16, int w16,
                                  float* __restrict__ out) {
  mivos::pdl_prologue();
  const int H = h16 * 16, W = w16 * 16;
  const int64_t total = 2ll * H * W;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % W);
    const int64_t t1 = i / W;
    const int y = static_cast<int>(t1 % H);
    const int pl = static_cast<int>(t1 / H);
    float sy = 0.0625f * (static_cast<float>(y) + 0.5f) - 0.5f;
    float sx = 0.0625f * (static_cast<float>(x) + 0.5f) - 0.5f;
    if (sy < 0.f) sy = 0.f;
    if (sx < 0.f) sx = 0.f;
    const int y0 = static_cast<int>(sy), x0 = static_cast<int>(sx);
    const int y1 = y0 + (y0 < h16 - 1 ? 1 : 0), x1 = x0 + (x0 < w16 - 1 ? 1 : 0);
    const float ly = sy - y0, lx = sx - x0, hy = 1.f - ly, hx = 1.f - lx;
    const float* m = maps + static_cast<int64_t>(pl) * h16 * w16;
    out[i] = hy * (hx * m[y0 * w16 + x0] + lx * m[y0 * w16 + x1]) +
             ly * (hx * m[y1 * w16 + x0] + lx * m[y1 * w16 + x1]);
  }
}

// Dynamic shared memory of attention_kernel: the query tile plus one logit row per query.
constexpr int kMaxAttentionSmem = 220 * 1024;  // hw <= 6912
inline int64_t attention_smem(int64_t hw) { return (QB * 128 + QB * hw) * 4; }

// Both entry points launch attention_kernel, so they share one record of its opt-in limit.  The
// attribute is only ever raised: lowering it for a smaller request would make a later launch of a
// size in between fail, since that size had already been allowed.
std::mutex g_attention_smem_mu;
int g_attention_smem = 0;

cudaError_t reserve_attention_smem(int smem) {
  std::lock_guard<std::mutex> lock(g_attention_smem_mu);
  if (smem <= g_attention_smem) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e == cudaSuccess) g_attention_smem = smem;
  return e;
}

// ------------------------------------------------------------------------------------------
// Streamed attention: the same softmax over the memory axis for ANY hw.  attention_kernel keeps a
// whole logit column per query in shared memory (hw <= 6912, below a 1080p frame's 8160 key pixels);
// here a CTA keeps only its SQ query rows qk/sqrt(128) resident and streams mk through shared memory
// SK keys at a time.  Warp w owns queries 4w..4w+3 of the CTA, lane l keys l, l+32, l+64, l+96 of the
// tile: the 4x4 logits of a thread are fp32 fma chains over the channels in ascending order, the
// chain of attention_kernel (the same bits).  The softmax is ONLINE (one pass): per tile the warp
// takes the tile maximum m_t, every lane rescales its partial sums by fl(expf(m - max(m, m_t))) —
// exactly 1 when the running maximum holds — and adds expf(s - max(m, m_t)).  The final maximum
// equals attention_kernel's (max is exact).
//   MODE 0  map:   maps[p][j] = sum_i e_ij pooled[p][i] / sum_i e_ij
//   MODE 1  stats: stats[j] = max_i s_ij, stats[hw + j] = sum_i expf(s_ij - max) (online, as MODE 0)
//   MODE 2  W:     w_out[i][j] = expf(s_ij - stats[j]) / stats[hw + j]; the tile is transposed through
//                  shared memory so that every warp store is one 128-byte run of a W row.
constexpr int SQ = 32;         // queries per CTA
constexpr int SK = 128;        // keys per shared-memory tile
constexpr int SK_PITCH = 132;  // floats per staged key row: the 8 rows of a quarter-warp's 16-byte loads hit 8 bank quads
constexpr int STREAM_THREADS = 256;
constexpr int kStreamSmem = (SQ * 128 + SK * SK_PITCH + 2 * SK) * 4;  // 84992 B: query rows, key tile, pooled tile
static_assert(SK * (SQ + 1) <= SK * SK_PITCH, "the W tile reuses the key tile");

template <int MODE>
__global__ void __launch_bounds__(STREAM_THREADS)
attention_stream_kernel(const float* __restrict__ mk, const float* __restrict__ qk, int hw,
                        const float* __restrict__ pooled, float* __restrict__ maps, float* __restrict__ stats,
                        float* __restrict__ w_out) {
  mivos::pdl_prologue();
  extern __shared__ __align__(16) float sm[];
  float* qs = sm;                  // [SQ][128]
  float* ks = qs + SQ * 128;       // [SK][SK_PITCH]; MODE 2: then the W tile [SK][SQ + 1]
  float* ps = ks + SK * SK_PITCH;  // [2][SK] pooled pos / neg of the tile's keys (MODE 0)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int j0 = blockIdx.x * SQ;
  for (int i = tid; i < SQ * 128; i += STREAM_THREADS) {
    const int q = i >> 7, c = i & 127;
    qs[i] = (j0 + q < hw) ? qk[static_cast<int64_t>(j0 + q) * 128 + c] / kSqrtCK : 0.f;
  }
  float m[4], den[4], pp[4], nn[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int j = j0 + warp * 4 + q;
    m[q] = MODE == 2 ? (j < hw ? stats[j] : 0.f) : -INFINITY;
    den[q] = MODE == 2 ? (j < hw ? stats[hw + j] : 1.f) : 0.f;
    pp[q] = nn[q] = 0.f;
  }
  for (int t0 = 0; t0 < hw; t0 += SK) {
    __syncthreads();  // the previous tile (or the W tile over it) has been consumed
    for (int i = tid; i < SK * 32; i += STREAM_THREADS) {
      const int r = i >> 5, c4 = i & 31;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t0 + r < hw) v = reinterpret_cast<const float4*>(mk + static_cast<int64_t>(t0 + r) * 128)[c4];
      *reinterpret_cast<float4*>(ks + r * SK_PITCH + c4 * 4) = v;
    }
    if (MODE == 0)
      for (int i = tid; i < 2 * SK; i += STREAM_THREADS) {
        const int p = i / SK, r = i - p * SK;
        ps[i] = t0 + r < hw ? pooled[static_cast<int64_t>(p) * hw + t0 + r] : 0.f;
      }
    __syncthreads();
    float s[4][4];  // [query q][key lane + 32 r]
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int r = 0; r < 4; ++r) s[q][r] = 0.f;
#pragma unroll 4
    for (int c4 = 0; c4 < 32; ++c4) {
      float4 kv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) kv[r] = *reinterpret_cast<const float4*>(ks + (lane + 32 * r) * SK_PITCH + c4 * 4);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 qv = *reinterpret_cast<const float4*>(qs + (warp * 4 + q) * 128 + c4 * 4);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          s[q][r] = fmaf(kv[r].x, qv.x, s[q][r]);
          s[q][r] = fmaf(kv[r].y, qv.y, s[q][r]);
          s[q][r] = fmaf(kv[r].z, qv.z, s[q][r]);
          s[q][r] = fmaf(kv[r].w, qv.w, s[q][r]);
        }
      }
    }
    if constexpr (MODE == 2) {
      __syncthreads();  // every warp is done with the key tile: it becomes the W tile
      float* wt = ks;
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int r = 0; r < 4; ++r) wt[(lane + 32 * r) * (SQ + 1) + warp * 4 + q] = expf(s[q][r] - m[q]) / den[q];
      __syncthreads();
      const int nq = hw - j0 < SQ ? hw - j0 : SQ;
      for (int r = warp; r < SK && t0 + r < hw; r += STREAM_THREADS / 32)
        if (lane < nq) w_out[static_cast<int64_t>(t0 + r) * hw + j0 + lane] = wt[r * (SQ + 1) + lane];
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float tmax = -INFINITY;
#pragma unroll
        for (int r = 0; r < 4; ++r)
          if (t0 + lane + 32 * r < hw) tmax = fmaxf(tmax, s[q][r]);
        const float mn = fmaxf(m[q], warp_max(tmax));
        const float c = expf(m[q] - mn);  // 0 on the first tile (m = -inf)
        m[q] = mn;
        den[q] *= c;
        if (MODE == 0) {
          pp[q] *= c;
          nn[q] *= c;
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          if (t0 + lane + 32 * r >= hw) continue;
          const float e = expf(s[q][r] - mn);
          den[q] += e;
          if (MODE == 0) {
            pp[q] = fmaf(e, ps[lane + 32 * r], pp[q]);
            nn[q] = fmaf(e, ps[SK + lane + 32 * r], nn[q]);
          }
        }
      }
    }
  }
  if constexpr (MODE != 2) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + warp * 4 + q;
      const float d = warp_sum(den[q]);
      const float p = MODE == 0 ? warp_sum(pp[q]) : 0.f;
      const float n = MODE == 0 ? warp_sum(nn[q]) : 0.f;
      if (lane == 0 && j < hw) {
        if (MODE == 0) {
          maps[j] = p / d;
          maps[hw + j] = n / d;
        } else {
          stats[j] = m[q];
          stats[hw + j] = d;
        }
      }
    }
  }
}

// The streamed kernels' opt-in shared-memory limit: one fixed size, set once per process (a record of its own:
// attention_kernel's record above is never touched).
std::mutex g_stream_smem_mu;
bool g_stream_smem_set = false;

cudaError_t reserve_stream_smem() {
  std::lock_guard<std::mutex> lock(g_stream_smem_mu);
  if (g_stream_smem_set) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(attention_stream_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStreamSmem);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(attention_stream_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStreamSmem);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(attention_stream_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStreamSmem);
  g_stream_smem_set = e == cudaSuccess;
  return e;
}

// Largest hw the streamed entry points take: 2·hw pooled cells and the launch grids stay in int range.
constexpr int64_t kMaxStreamHw = int64_t{1} << 28;

}  // namespace
}  // namespace mivos

using namespace mivos;

extern "C" MIVOS_API int mivos_attention_map(const float* mk, const float* qk, int h16, int w16,
                                             const float* pos, const float* neg, float* out,
                                             float* scratch, mivos_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MIVOS_REQUIRE(mk && qk && pos && neg && out && scratch, "attention_map: null pointer");
  MIVOS_REQUIRE((reinterpret_cast<uintptr_t>(mk) & 15) == 0 && (reinterpret_cast<uintptr_t>(qk) & 15) == 0,
                "attention_map: mk/qk must be 16-byte aligned");
  MIVOS_REQUIRE(h16 > 0 && w16 > 0, "attention_map: bad key grid %d x %d", h16, w16);
  MIVOS_REQUIRE(attention_smem(static_cast<int64_t>(h16) * w16) <= kMaxAttentionSmem,
                "attention_map: %d x %d key pixels exceed the shared-memory tile", h16, w16);
  const int hw = h16 * w16;
  const int smem = static_cast<int>(attention_smem(hw));
  // scratch: pooled[2][hw] followed by maps[2][hw]
  float* pooled = scratch;
  float* maps = scratch + 2 * hw;
  launch_pdl(area_pool16_kernel, ceil_div(2 * hw, 128), 128, 0, stream, pos, neg, h16, w16, pooled);
  g_launches.fetch_add(1);
  MIVOS_CUDA_OK(cudaGetLastError());
  MIVOS_CUDA_OK(reserve_attention_smem(smem));
  launch_pdl(attention_kernel, ceil_div(hw, QB), ATT_THREADS, smem, stream, mk, qk, hw, pooled, maps,
             static_cast<float*>(nullptr));
  g_launches.fetch_add(1);
  MIVOS_CUDA_OK(cudaGetLastError());
  const int64_t total = 2ll * hw * 256;
  int64_t g = (total + 255) / 256;
  if (g > num_sms() * 16) g = num_sms() * 16;
  launch_pdl(upsample16_kernel, static_cast<unsigned>(g), 256, 0, stream, maps, h16, w16, out);
  g_launches.fetch_add(1);
  MIVOS_CUDA_OK(cudaGetLastError());
  return MIVOS_OK;
}

// PropagationNetwork.get_W / AttentionMemory.forward (prop_net.py:115-129,183): W[i, j] =
// softmax over memory pixels i of mk[i] . qk[j] / sqrt(128), written out as [hw, hw] fp32.
// `scratch` (4*hw floats, as for mivos_attention_map) receives throw-away reductions.
extern "C" MIVOS_API int mivos_attention_weights(const float* mk, const float* qk, int hw, float* w_out,
                                                 float* scratch, mivos_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MIVOS_REQUIRE(mk && qk && w_out && scratch, "attention_weights: null pointer");
  MIVOS_REQUIRE((reinterpret_cast<uintptr_t>(mk) & 15) == 0 && (reinterpret_cast<uintptr_t>(qk) & 15) == 0,
                "attention_weights: mk/qk must be 16-byte aligned");
  MIVOS_REQUIRE(hw > 0 && attention_smem(hw) <= kMaxAttentionSmem,
                "attention_weights: %d key pixels exceed the shared-memory tile", hw);
  const int smem = static_cast<int>(attention_smem(hw));
  MIVOS_CUDA_OK(cudaMemsetAsync(scratch, 0, static_cast<size_t>(2) * hw * 4, stream));  // pooled = 0: maps unused
  MIVOS_CUDA_OK(reserve_attention_smem(smem));
  launch_pdl(attention_kernel, ceil_div(hw, QB), ATT_THREADS, smem, stream, mk, qk, hw, scratch, scratch + 2 * hw, w_out);
  g_launches.fetch_add(1);
  MIVOS_CUDA_OK(cudaGetLastError());
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_attention_plan(int hw, int* resident) {
  MIVOS_REQUIRE(resident, "attention_plan: null pointer");
  MIVOS_REQUIRE(hw > 0, "attention_plan: %d key pixels", hw);
  *resident = attention_smem(hw) <= kMaxAttentionSmem ? 1 : 0;
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_attention_map_streamed(const float* mk, const float* qk, int h16, int w16,
                                                      const float* pos, const float* neg, float* out, float* scratch,
                                                      mivos_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MIVOS_REQUIRE(mk && qk && pos && neg && out && scratch, "attention_map_streamed: null pointer");
  MIVOS_REQUIRE((reinterpret_cast<uintptr_t>(mk) & 15) == 0 && (reinterpret_cast<uintptr_t>(qk) & 15) == 0,
                "attention_map_streamed: mk/qk must be 16-byte aligned");
  MIVOS_REQUIRE(h16 > 0 && w16 > 0 && static_cast<int64_t>(h16) * w16 <= kMaxStreamHw,
                "attention_map_streamed: bad key grid %d x %d", h16, w16);
  const int hw = h16 * w16;
  // scratch: pooled[2][hw] followed by maps[2][hw]
  float* pooled = scratch;
  float* maps = scratch + 2 * static_cast<int64_t>(hw);
  MIVOS_CUDA_OK(reserve_stream_smem());
  launch_pdl(area_pool16_kernel, ceil_div(2 * hw, 128), 128, 0, stream, pos, neg, h16, w16, pooled);
  g_launches.fetch_add(1);
  MIVOS_CUDA_OK(cudaGetLastError());
  launch_pdl(attention_stream_kernel<0>, ceil_div(hw, SQ), STREAM_THREADS, kStreamSmem, stream, mk, qk, hw, pooled,
             maps, static_cast<float*>(nullptr), static_cast<float*>(nullptr));
  g_launches.fetch_add(1);
  MIVOS_CUDA_OK(cudaGetLastError());
  const int64_t total = 2ll * hw * 256;
  int64_t g = (total + 255) / 256;
  if (g > num_sms() * 16) g = num_sms() * 16;
  launch_pdl(upsample16_kernel, static_cast<unsigned>(g), 256, 0, stream, maps, h16, w16, out);
  g_launches.fetch_add(1);
  MIVOS_CUDA_OK(cudaGetLastError());
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_attention_weights_streamed(const float* mk, const float* qk, int hw, float* w_out,
                                                          float* scratch, mivos_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MIVOS_REQUIRE(mk && qk && w_out && scratch, "attention_weights_streamed: null pointer");
  MIVOS_REQUIRE((reinterpret_cast<uintptr_t>(mk) & 15) == 0 && (reinterpret_cast<uintptr_t>(qk) & 15) == 0,
                "attention_weights_streamed: mk/qk must be 16-byte aligned");
  MIVOS_REQUIRE(hw > 0 && hw <= kMaxStreamHw, "attention_weights_streamed: %d key pixels", hw);
  // scratch: per query column the maximum [hw] and the denominator [hw]
  MIVOS_CUDA_OK(reserve_stream_smem());
  const float* none = nullptr;
  launch_pdl(attention_stream_kernel<1>, ceil_div(hw, SQ), STREAM_THREADS, kStreamSmem, stream, mk, qk, hw, none,
             static_cast<float*>(nullptr), scratch, static_cast<float*>(nullptr));
  g_launches.fetch_add(1);
  MIVOS_CUDA_OK(cudaGetLastError());
  launch_pdl(attention_stream_kernel<2>, ceil_div(hw, SQ), STREAM_THREADS, kStreamSmem, stream, mk, qk, hw, none,
             static_cast<float*>(nullptr), scratch, w_out);
  g_launches.fetch_add(1);
  MIVOS_CUDA_OK(cudaGetLastError());
  return MIVOS_OK;
}
