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
