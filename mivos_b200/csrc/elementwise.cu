// HBM-bound kernels of the propagation path: gathers that feed the implicit GEMM, pooling,
// bilinear resampling, layout conversion at the API boundary, soft aggregation and argmax.
// All are coalesced / 128-bit vectorised streaming kernels; none has data reuse worth staging
// beyond the transposes (which go through a padded shared-memory tile).
#include "groups.cuh"
#include "host_util.h"
#include "pdl.cuh"

#include <atomic>

namespace mivos {
extern std::atomic<int64_t> g_launches;
namespace {

constexpr int kThreads = 256;

#define MIVOS_LAUNCHED()                                   \
  do {                                                     \
    g_launches.fetch_add(1, std::memory_order_relaxed);    \
    MIVOS_CUDA_OK(cudaGetLastError());                     \
  } while (0)

// ------------------------------------------------------------------------------------------
// bilinear source index, align_corners=False (ATen area_pixel_compute_source_index)
__device__ __forceinline__ void bilin(int dst, float scale, int in_size, int& i0, int& i1, float& l1) {
  float src = scale * (static_cast<float>(dst) + 0.5f) - 0.5f;
  if (src < 0.f) src = 0.f;
  i0 = static_cast<int>(src);
  i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
  l1 = src - static_cast<float>(i0);
}

// ------------------------------------------------------------------------------------------
// SETS: set s (per_set consecutive objects) writes bank frame dyn_t[s]; a frame outside [0, t] writes nothing.
// GROUPS (with SETS): the set of an object is its group in `first` (groups.cuh); an object in no group writes nothing.
template <bool SETS, bool GROUPS = false>
__global__ void bank_write_kernel(const float4* __restrict__ halo, int kobj, int h, int w,
                                  int cstride4, int coffk4, int coffv4, float4* __restrict__ bank_k,
                                  float4* __restrict__ bank_v, int64_t slots_cap, int t,
                                  const int* __restrict__ dyn_t, int per_set, const int* __restrict__ first,
                                  int groups) {
  mivos::pdl_prologue();
  const int t_max = t;
  if (!SETS && dyn_t) t = *dyn_t;  // bank slot from device memory (CUDA-graph replay)
  const int hw = h * w;
  const int per_pix = 32 + 128;  // float4s of key + value
  const int64_t total = static_cast<int64_t>(kobj) * hw * per_pix;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int e = static_cast<int>(i % per_pix);
    const int64_t t1 = i / per_pix;
    const int p = static_cast<int>(t1 % hw);
    const int obj = static_cast<int>(t1 / hw);
    if (SETS) {
      const int s = GROUPS ? map_group(first, groups, kobj, obj) : obj / per_set;
      if (GROUPS && s < 0) continue;
      t = dyn_t[s];
      if (t < 0 || t > t_max) continue;
    }
    const int y = p / w, x = p - y * w;
    const int64_t r = (static_cast<int64_t>(obj) * (h + 2) + y + 1) * (w + 2) + x + 1;
    const int64_t slot = static_cast<int64_t>(t) * hw + p;
    if (e < 32) {
      bank_k[(static_cast<int64_t>(obj) * slots_cap + slot) * 32 + e] = halo[r * cstride4 + coffk4 + e];
    } else {
      bank_v[(static_cast<int64_t>(obj) * slots_cap + slot) * 128 + (e - 32)] = halo[r * cstride4 + coffv4 + (e - 32)];
    }
  }
}

// src [obj][C][slots] -> dst [obj][slots_cap][C]; grid (slot tiles, C tiles, obj)
__global__ void bank_transpose_kernel(const float* __restrict__ src, int c, int64_t slots,
                                      float* __restrict__ dst, int64_t slots_cap) {
  mivos::pdl_prologue();
  __shared__ float tile[32][33];
  const int obj = blockIdx.z;
  const int64_t s0 = static_cast<int64_t>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int j = ty; j < 32; j += 8) {
    const int ch = c0 + j;
    const int64_t s = s0 + tx;
    tile[j][tx] = (s < slots && ch < c) ? src[(static_cast<int64_t>(obj) * c + ch) * slots + s] : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int64_t s = s0 + j;
    const int ch = c0 + tx;
    if (s < slots && ch < c) dst[(static_cast<int64_t>(obj) * slots_cap + s) * c + ch] = tile[tx][j];
  }
}

// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf_exact(float x) { return 1.f / (1.f + expf(-x)); }

constexpr int kMaxObjects = 16;

// aggregate_wbg (aggregate.py:22-37) for one pixel: p[0..k) object probabilities in, softmax of
// logit(clamp([prod(1-p), p...])) out (o[0] = background).
__device__ __forceinline__ void aggregate_pixel(const float* p, int k, bool hard, float* o,
                                                bool const_bg = false) {
  float bg = 1.f;
  for (int j = 0; j < k; ++j) bg *= (1.f - p[j]);
  if (const_bg) bg = 0.5f;  // aggregate_sbg (aggregate.py:8)
  float mx = -INFINITY;
  for (int j = 0; j <= k; ++j) {
    float v = (j == 0) ? bg : p[j - 1];
    v = fminf(fmaxf(v, 1e-7f), 1.f - 1e-7f);
    float l = logf(v / (1.f - v));
    if (hard) l *= 1000.f;
    o[j] = l;
    mx = fmaxf(mx, l);
  }
  float s = 0.f;
  for (int j = 0; j <= k; ++j) {
    o[j] = expf(o[j] - mx);
    s += o[j];
  }
  for (int j = 0; j <= k; ++j) o[j] = o[j] / s;
}

// GROUPS: group g is maps [first[g], first[g+1]) of `kobj` maps (groups.cuh), its planes start at first[g] in
// raw_out and at first[g] + g in prob_out (packed: each group's background plane, then its objects); a group that is
// empty, outside [0, kobj] or of more than kMaxObjects maps writes nothing.
template <bool GROUPS>
__global__ void upsample4x_sigmoid_aggregate_kernel(const float* __restrict__ logits_all, int kobj,
                                                    int h4, int w4, int cstride, int coff,
                                                    float* __restrict__ raw_all,
                                                    float* __restrict__ prob_all, int groups,
                                                    const int* __restrict__ first) {
  mivos::pdl_prologue();
  const int H = 4 * h4, W = 4 * w4;
  const int64_t plane = static_cast<int64_t>(H) * W;
  // group g (a clip of a lock-step step) = images [g*kobj, (g+1)*kobj) of the logits, planes
  // [g*kobj, ...) of raw_out and [g*(kobj+1), ...) of prob_out; the aggregation runs within a group
  for (int64_t ig = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; ig < plane * groups;
       ig += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(ig / plane);
    const int64_t i = ig - static_cast<int64_t>(g) * plane;
    int m0 = g * kobj, k = kobj;
    if (GROUPS && (!group_range(first, kobj, g, &m0, &k) || k > kMaxObjects)) continue;
    const int64_t p0 = GROUPS ? m0 + g : static_cast<int64_t>(g) * (kobj + 1);
    const float* logits = logits_all + static_cast<int64_t>(m0) * (h4 + 2) * (w4 + 2) * cstride;
    float* raw_out = raw_all ? raw_all + static_cast<int64_t>(m0) * plane : nullptr;
    float* prob_out = prob_all ? prob_all + p0 * plane : nullptr;
    const int y = static_cast<int>(i / W), x = static_cast<int>(i - static_cast<int64_t>(y) * W);
    int y0, y1, x0, x1;
    float ly, lx;
    bilin(y, 0.25f, h4, y0, y1, ly);
    bilin(x, 0.25f, w4, x0, x1, lx);
    const float hy = 1.f - ly, hx = 1.f - lx;
    float p[kMaxObjects], o[kMaxObjects + 1];
    for (int j = 0; j < k; ++j) {
      const int64_t base = static_cast<int64_t>(j) * (h4 + 2);
      const float v00 = logits[((base + y0 + 1) * (w4 + 2) + x0 + 1) * cstride + coff];
      const float v01 = logits[((base + y0 + 1) * (w4 + 2) + x1 + 1) * cstride + coff];
      const float v10 = logits[((base + y1 + 1) * (w4 + 2) + x0 + 1) * cstride + coff];
      const float v11 = logits[((base + y1 + 1) * (w4 + 2) + x1 + 1) * cstride + coff];
      const float v = hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11);
      p[j] = sigmoidf_exact(v);
      if (raw_out) raw_out[j * plane + i] = p[j];
    }
    if (prob_out) {
      aggregate_pixel(p, k, false, o);
      for (int j = 0; j <= k; ++j) prob_out[j * plane + i] = o[j];
    }
  }
}

// ---- aggregation over any object count (mivos_*_planes).  The kernels above hold a pixel's K values in
// per-thread arrays of kMaxObjects; these hold none: the object values live in planes in global memory and a
// thread makes passes over them — background product, logits (written over the planes) and their maximum,
// exponentials (written over the logits) and their sum, normalisation — in the operation order of
// aggregate_pixel, so for K <= 16 they give its bits.
__device__ __forceinline__ float clamped_logit(float v, bool hard) {
  v = fminf(fmaxf(v, 1e-7f), 1.f - 1e-7f);
  float l = logf(v / (1.f - v));
  if (hard) l *= 1000.f;
  return l;
}

// Group g, pixel i: object j at in[g*in_gstride + j*plane + i]; the result at out[g*out_gstride + ...], background
// first when keep_bg.  `in` may be the object planes of `out` itself (in place: in == out + plane, keep_bg).
__global__ void aggregate_planes_kernel(const float* in, int kobj, int64_t plane, int groups, int64_t in_gstride,
                                        float* out, int64_t out_gstride, int keep_bg, int hard) {
  mivos::pdl_prologue();
  const bool hl = (hard & 1) != 0;
  for (int64_t ig = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; ig < plane * groups;
       ig += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t g = ig / plane, i = ig - g * plane;
    const float* p = in + g * in_gstride + i;
    float* o = out + g * out_gstride + i;
    float* ob = keep_bg ? o + plane : o;  // object j of the result at ob[j * plane]
    float bg = 1.f;
    if (hard & 2) {
      bg = 0.5f;  // aggregate_sbg (aggregate.py:8)
    } else {
      for (int j = 0; j < kobj; ++j) bg *= (1.f - p[j * plane]);
    }
    const float l0 = clamped_logit(bg, hl);
    float mx = l0;
    for (int j = 0; j < kobj; ++j) {
      const float l = clamped_logit(p[j * plane], hl);
      ob[j * plane] = l;
      mx = fmaxf(mx, l);
    }
    const float e0 = expf(l0 - mx);
    float s = e0;
    for (int j = 0; j < kobj; ++j) {
      const float e = expf(ob[j * plane] - mx);
      ob[j * plane] = e;
      s += e;
    }
    if (keep_bg) o[0] = e0 / s;
    for (int j = 0; j < kobj; ++j) ob[j * plane] = ob[j * plane] / s;
  }
}

// x4 bilinear + sigmoid of every object map, one thread per (image, pixel): image g*kobj + j of the logits to
// raw_all[(g*kobj + j)*plane] and/or obj_all[g*obj_gstride + j*plane] (the object planes of a prob volume).
__global__ void upsample4x_sigmoid_planes_kernel(const float* __restrict__ logits, int kobj, int h4, int w4,
                                                 int cstride, int coff, int groups, float* __restrict__ raw_all,
                                                 float* __restrict__ obj_all, int64_t obj_gstride) {
  mivos::pdl_prologue();
  const int H = 4 * h4, W = 4 * w4;
  const int64_t plane = static_cast<int64_t>(H) * W;
  const int64_t total = plane * kobj * groups;
  for (int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t img = t / plane, i = t - img * plane;
    const int y = static_cast<int>(i / W), x = static_cast<int>(i - static_cast<int64_t>(y) * W);
    int y0, y1, x0, x1;
    float ly, lx;
    bilin(y, 0.25f, h4, y0, y1, ly);
    bilin(x, 0.25f, w4, x0, x1, lx);
    const float hy = 1.f - ly, hx = 1.f - lx;
    const int64_t base = img * (h4 + 2);
    const float v00 = logits[((base + y0 + 1) * (w4 + 2) + x0 + 1) * cstride + coff];
    const float v01 = logits[((base + y0 + 1) * (w4 + 2) + x1 + 1) * cstride + coff];
    const float v10 = logits[((base + y1 + 1) * (w4 + 2) + x0 + 1) * cstride + coff];
    const float v11 = logits[((base + y1 + 1) * (w4 + 2) + x1 + 1) * cstride + coff];
    // the roundings the compiler picks for the same expression in upsample4x_sigmoid_aggregate_kernel, spelled out
    const float v = __fmaf_rn(hy, __fmaf_rn(hx, v00, __fmul_rn(lx, v01)), __fmul_rn(ly, __fmaf_rn(hx, v10, __fmul_rn(lx, v11))));
    const float p = sigmoidf_exact(v);
    if (raw_all) raw_all[t] = p;
    if (obj_all) {
      const int64_t g = img / kobj, j = img - g * kobj;
      obj_all[g * obj_gstride + j * plane + i] = p;
    }
  }
}

// bilinear resize (align_corners=False, any ratio) of ONE channel of a HALO map to NCHW planes
// [n,1,H,W], optionally through a sigmoid: the final F.interpolate of the S2M network
// (model/s2m/utils.py:20) and the torch.sigmoid its callers apply (davis_processor.py:68,
// interact/s2m_controller.py:35).
__global__ void halo_upsample_to_plane_kernel(const float* __restrict__ halo, int n, int hs, int ws, int cstride,
                                              int coff, int H, int W, float sy, float sx, int sigmoid,
                                              float* __restrict__ out) {
  mivos::pdl_prologue();
  const int64_t plane = static_cast<int64_t>(H) * W;
  const int64_t total = plane * n;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int img = static_cast<int>(i / plane);
    const int64_t pi = i - static_cast<int64_t>(img) * plane;
    const int y = static_cast<int>(pi / W), x = static_cast<int>(pi - static_cast<int64_t>(y) * W);
    int y0, y1, x0, x1;
    float ly, lx;
    bilin(y, sy, hs, y0, y1, ly);
    bilin(x, sx, ws, x0, x1, lx);
    const float hy = 1.f - ly, hx = 1.f - lx;
    const int64_t base = static_cast<int64_t>(img) * (hs + 2);
    const float v00 = halo[((base + y0 + 1) * (ws + 2) + x0 + 1) * cstride + coff];
    const float v01 = halo[((base + y0 + 1) * (ws + 2) + x1 + 1) * cstride + coff];
    const float v10 = halo[((base + y1 + 1) * (ws + 2) + x0 + 1) * cstride + coff];
    const float v11 = halo[((base + y1 + 1) * (ws + 2) + x1 + 1) * cstride + coff];
    const float v = hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11);
    out[i] = sigmoid ? sigmoidf_exact(v) : v;
  }
}

// overlay_davis / overlay_davis_fade (interact/interactive_utils.py:119-143): the GUI's per-frame
// display composite.  image u8 [t][h][w][3], mask u8 [t][h][w], colors u8 [ncolors][3].
//   labelled pixel      : trunc(image * alpha + (1 - alpha) * colors[label])   (float64 like numpy,
//                         separately rounded products: no FMA contraction)
//   4-connected contour : 0      (binary_dilation(mask > 0) ^ (mask > 0), border value 0)
//   other pixels        : image  (fade: trunc(image * 0.6))
// One thread per pixel; HBM-bound: 4 B read + 3 B written per pixel (neighbour labels hit L1/L2).
__global__ void overlay_davis_kernel(const uint8_t* __restrict__ image, const uint8_t* __restrict__ mask, int t, int h,
                                     int w, const uint8_t* __restrict__ colors, int ncolors, double alpha, int fade,
                                     uint8_t* __restrict__ out) {
  mivos::pdl_prologue();
  const int64_t plane = static_cast<int64_t>(h) * w;
  const int64_t total = plane * t;
  const double beta = 1.0 - alpha;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t pi = i % plane;
    const int y = static_cast<int>(pi / w), x = static_cast<int>(pi - static_cast<int64_t>(y) * w);
    const int m = mask[i];
    const uint8_t* px = image + i * 3;
    uint8_t o[3] = {px[0], px[1], px[2]};
    if (m > 0) {
      const int ci = m < ncolors ? m : 0;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double v = __dadd_rn(__dmul_rn(static_cast<double>(px[c]), alpha), __dmul_rn(beta, static_cast<double>(colors[ci * 3 + c])));
        o[c] = static_cast<uint8_t>(static_cast<int>(v));
      }
    } else {
      const bool contour = (y > 0 && mask[i - w] > 0) || (y + 1 < h && mask[i + w] > 0) || (x > 0 && mask[i - 1] > 0) ||
                           (x + 1 < w && mask[i + 1] > 0);
      if (contour) {
        o[0] = o[1] = o[2] = 0;
      } else if (fade) {
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c] = static_cast<uint8_t>(static_cast<int>(__dmul_rn(static_cast<double>(px[c]), 0.6)));
      }
    }
    out[i * 3] = o[0];
    out[i * 3 + 1] = o[1];
    out[i * 3 + 2] = o[2];
  }
}

__global__ void aggregate_wbg_kernel(const float* __restrict__ prob, int kobj, int64_t hw,
                                     int keep_bg, int hard, float* __restrict__ out) {
  mivos::pdl_prologue();
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < hw;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float p[kMaxObjects], o[kMaxObjects + 1];
    for (int j = 0; j < kobj; ++j) p[j] = prob[j * hw + i];
    aggregate_pixel(p, kobj, (hard & 1) != 0, o, (hard & 2) != 0);
    if (keep_bg) {
      for (int j = 0; j <= kobj; ++j) out[j * hw + i] = o[j];
    } else {
      for (int j = 1; j <= kobj; ++j) out[(j - 1) * hw + i] = o[j];
    }
  }
}

// prob [(K+1)][T][nh*nw] -> masks_padded [T][nh*nw] u8, masks_out [T][h][w] u8 (first max wins)
__global__ void argmax_unpad_kernel(const float* __restrict__ prob, int k1, int t, int nh, int nw,
                                    int pad_l, int pad_t, int h, int w,
                                    uint8_t* __restrict__ masks_padded,
                                    uint8_t* __restrict__ masks_out) {
  mivos::pdl_prologue();
  const int64_t plane = static_cast<int64_t>(nh) * nw;
  const int64_t total = static_cast<int64_t>(t) * plane;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float best = prob[i];
    int arg = 0;
    for (int j = 1; j < k1; ++j) {
      const float v = prob[static_cast<int64_t>(j) * total + i];
      if (v > best) { best = v; arg = j; }
    }
    masks_padded[i] = static_cast<uint8_t>(arg);
    if (masks_out) {
      const int ti = static_cast<int>(i / plane);
      const int rem = static_cast<int>(i - ti * plane);
      const int y = rem / nw - pad_t, x = rem % nw - pad_l;
      if (y >= 0 && y < h && x >= 0 && x < w)
        masks_out[(static_cast<int64_t>(ti) * h + y) * w + x] = static_cast<uint8_t>(arg);
    }
  }
}

__global__ void pad2d_kernel(const float* __restrict__ in, int planes, int h, int w, int pad_l,
                             int pad_t, int nh, int nw, float* __restrict__ out) {
  mivos::pdl_prologue();
  const int64_t total = static_cast<int64_t>(planes) * nh * nw;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % nw) - pad_l;
    const int64_t t1 = i / nw;
    const int y = static_cast<int>(t1 % nh) - pad_t;
    const int64_t pl = t1 / nh;
    float v = 0.f;
    if (y >= 0 && y < h && x >= 0 && x < w) v = in[(pl * h + y) * w + x];
    out[i] = v;
  }
}

__global__ void halo_sigmoid_to_plane_kernel(const float* __restrict__ halo, int h, int w,
                                             int cstride, int coff, float* __restrict__ plane) {
  mivos::pdl_prologue();
  const int64_t total = static_cast<int64_t>(h) * w;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / w), x = static_cast<int>(i - static_cast<int64_t>(y) * w);
    plane[i] = sigmoidf_exact(halo[(static_cast<int64_t>(y + 1) * (w + 2) + x + 1) * cstride + coff]);
  }
}

__global__ void halo_to_pixels_kernel(const float4* __restrict__ halo, int n, int h, int w, int cs4,
                                      int co4, int c4, float4* __restrict__ out) {
  mivos::pdl_prologue();
  const int64_t total = static_cast<int64_t>(n) * h * w * c4;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % c4);
    int64_t t1 = i / c4;
    const int x = static_cast<int>(t1 % w);
    t1 /= w;
    const int y = static_cast<int>(t1 % h);
    const int img = static_cast<int>(t1 / h);
    out[i] = halo[((static_cast<int64_t>(img) * (h + 2) + y + 1) * (w + 2) + x + 1) * cs4 + co4 + ci];
  }
}

// Frame ingest (interact/interactive_utils.py:18-23 images_to_torch; dataset/davis_test_dataset.py:49-52
// ToTensor + im_normalization): u8 HWC frames -> normalised fp32 planes, the same IEEE operations in
// the same order as `x.float() / 255` followed by torchvision's Normalize `(x - mean) / std`, so the
// result is bit-identical to the reference's CPU path.  One thread per pixel: a warp reads 96
// contiguous bytes and writes three coalesced 128-byte plane segments.
__global__ void frames_u8_normalize_kernel(const uint8_t* __restrict__ hwc, int64_t pixels_per_frame, int64_t total,
                                           float* __restrict__ out) {
  mivos::pdl_prologue();
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};  // dataset/range_transform.py:5-8
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t f = i / pixels_per_frame, pix = i - f * pixels_per_frame;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = __fdiv_rn(static_cast<float>(hwc[i * 3 + c]), 255.0f);
      out[(f * 3 + c) * pixels_per_frame + pix] = __fdiv_rn(__fsub_rn(v, mean[c]), stdv[c]);
    }
  }
}

__global__ void store_i32_kernel(int* dst, int n, int v0, int v1, int v2, int v3) {
  mivos::pdl_prologue();
  const int v[4] = {v0, v1, v2, v3};
  if (threadIdx.x < n) dst[threadIdx.x] = v[threadIdx.x];
}

// Per-frame words of a replayed CUDA graph, written from launch arguments (no host buffer to keep alive):
// up to 64 int64 (device pointers that change from frame to frame) and up to 4 int32 (bank counters).
struct StoreWords {
  int64_t v[64];
};
__global__ void store_words_kernel(int64_t* dst64, int n64, const StoreWords w, int* dst32, int n32, int v0, int v1,
                                   int v2, int v3) {
  mivos::pdl_prologue();
  const int t = threadIdx.x;
  if (t < n64) dst64[t] = w.v[t];
  const int v[4] = {v0, v1, v2, v3};
  if (t < n32) dst32[t] = v[t];
}

// Segment copies whose source OR destination pointer is read from device memory at run time (`dyn`), the other
// side and the byte counts being fixed when the launch was recorded: lets a captured graph stage per-frame
// operands (cached query features, the frame) and deliver its result (probability planes of frame ti) without
// eager copies between replays.  blockIdx.y = segment; 16-byte vectors; a null dyn pointer skips the segment.
__global__ void copy_segments_kernel(const int64_t* __restrict__ fixed, const int64_t* __restrict__ dyn,
                                     const int64_t* __restrict__ bytes, int dyn_is_src) {
  mivos::pdl_prologue();
  const int seg = blockIdx.y;
  const int64_t d = dyn[seg];
  if (d == 0) return;
  const uint4* src = reinterpret_cast<const uint4*>(dyn_is_src ? d : fixed[seg]);
  uint4* dst = reinterpret_cast<uint4*>(dyn_is_src ? fixed[seg] : d);
  const int64_t nvec = bytes[seg] >> 4;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = src[i];
}

// Result delivery to (host-mapped) volumes: blockIdx.y = clip, its record of MIVOS_DELIVER_WORDS words in `table`
// (header).  A thread owns 16 consecutive pixels of the padded plane: it reads each of the clip's K+1 planes once
// (four 16-byte loads), stores them to the volume in 16-byte stores (a warp writes 2 KB contiguous per plane) and
// keeps the running argmax, whose 16 labels go out as one 16-byte store.  The unpadded labels of the block's span
// go through shared memory so that consecutive threads store consecutive bytes of a row.
constexpr int kDeliverPix = 16;
constexpr int kDeliverSpan = kThreads * kDeliverPix;
__global__ void __launch_bounds__(kThreads) deliver_planes_kernel(const float* __restrict__ planes,
                                                                  const int64_t* __restrict__ table, int nh, int nw) {
  mivos::pdl_prologue();
  __shared__ uint8_t lab[kDeliverSpan];
  const int64_t* rec = table + static_cast<int64_t>(blockIdx.y) * MIVOS_DELIVER_WORDS;
  float* prob = reinterpret_cast<float*>(rec[0]);
  const int64_t stride = rec[1];
  uint8_t* lp = reinterpret_cast<uint8_t*>(rec[2]);
  uint8_t* lu = reinterpret_cast<uint8_t*>(rec[3]);
  const int src0 = static_cast<int>(rec[4] & 0xFFFFFFFF), k1 = static_cast<int>(rec[4] >> 32);
  const int pad_l = static_cast<int>(rec[5] & 0xFFFFFFFF), pad_t = static_cast<int>(rec[5] >> 32);
  const int h = static_cast<int>(rec[6] & 0xFFFFFFFF), w = static_cast<int>(rec[6] >> 32);
  if (prob == nullptr || k1 < 1 || k1 > MIVOS_MAX_OBJECTS + 1) return;  // uniform over the block
  const int64_t plane = static_cast<int64_t>(nh) * nw;
  const float* src = planes + static_cast<int64_t>(src0) * plane;
  for (int64_t base = static_cast<int64_t>(blockIdx.x) * kDeliverSpan; base < plane;
       base += static_cast<int64_t>(gridDim.x) * kDeliverSpan) {
    const int64_t i = base + threadIdx.x * kDeliverPix;
    if (i < plane) {
      float best[kDeliverPix];
      uint32_t arg[kDeliverPix / 4] = {0u, 0u, 0u, 0u};  // four labels per word, byte q%4 of word q/4
      for (int j = 0; j < k1; ++j) {
        const float4* s = reinterpret_cast<const float4*>(src + j * plane + i);
        float4* d = reinterpret_cast<float4*>(prob + j * stride + i);
#pragma unroll
        for (int v = 0; v < kDeliverPix / 4; ++v) {
          const float4 x = __ldg(s + v);
          d[v] = x;
          const float e[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int q = v * 4 + u;
            if (j == 0 || e[u] > best[q]) {
              best[q] = e[u];
              arg[v] = (arg[v] & ~(0xFFu << (8 * u))) | (static_cast<uint32_t>(j) << (8 * u));
            }
          }
        }
      }
      *reinterpret_cast<uint4*>(lp + i) = make_uint4(arg[0], arg[1], arg[2], arg[3]);
      *reinterpret_cast<uint4*>(lab + threadIdx.x * kDeliverPix) = make_uint4(arg[0], arg[1], arg[2], arg[3]);
    }
    __syncthreads();
    for (int q = threadIdx.x; q < kDeliverSpan && base + q < plane; q += kThreads) {
      const int64_t p = base + q;
      const int y = static_cast<int>(p / nw) - pad_t, x = static_cast<int>(p % nw) - pad_l;
      if (y >= 0 && y < h && x >= 0 && x < w) lu[static_cast<int64_t>(y) * w + x] = lab[q];
    }
    __syncthreads();
  }
}

inline unsigned capped_grid(int64_t work) {
  // grid-stride kernels: a few waves of the SMs x 8 resident 256-thread CTAs is plenty
  const int64_t cap = num_sms() * 16ll;
  int64_t g = (work + kThreads - 1) / kThreads;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<unsigned>(g);
}

}  // namespace
}  // namespace mivos

using namespace mivos;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define AL16(p) ((reinterpret_cast<uintptr_t>(p) & 15) == 0)

extern "C" MIVOS_API int mivos_bank_write(const float* halo, int k_objects, int h, int w, int cstride,
                                          int coff_k, int coff_v, float* bank_k, float* bank_v,
                                          int64_t slots_cap, int t, const int32_t* dyn_t, mivos_stream_t s) {
  MIVOS_REQUIRE(halo && bank_k && bank_v && AL16(halo) && AL16(bank_k) && AL16(bank_v), "bank_write: null/unaligned pointer");
  MIVOS_REQUIRE(cstride % 4 == 0 && coff_k % 4 == 0 && coff_v % 4 == 0 && t >= 0 &&
                    static_cast<int64_t>(t + 1) * h * w <= slots_cap,
                "bank_write: slot %d does not fit capacity %lld", t, (long long)slots_cap);
  const int64_t total = static_cast<int64_t>(k_objects) * h * w * 160;
  launch_pdl(bank_write_kernel<false>, capped_grid(total), kThreads, 0, ST(s), 
      reinterpret_cast<const float4*>(halo), k_objects, h, w, cstride / 4, coff_k / 4, coff_v / 4,
      reinterpret_cast<float4*>(bank_k), reinterpret_cast<float4*>(bank_v), slots_cap, t, dyn_t, 0, nullptr, 0);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_bank_write_sets(const float* halo, int k_objects, int sets, int h, int w, int cstride,
                                               int coff_k, int coff_v, float* bank_k, float* bank_v,
                                               int64_t slots_cap, int t_max, const int32_t* dyn_t, mivos_stream_t s) {
  MIVOS_REQUIRE(dyn_t, "bank_write_sets: null frame array (one device-side bank frame per set)");
  MIVOS_REQUIRE(sets >= 1 && k_objects >= 1 && k_objects % sets == 0, "bank_write_sets: %d sets do not divide %d objects",
                sets, k_objects);
  MIVOS_REQUIRE(halo && bank_k && bank_v && AL16(halo) && AL16(bank_k) && AL16(bank_v),
                "bank_write_sets: null/unaligned pointer");
  MIVOS_REQUIRE(cstride % 4 == 0 && coff_k % 4 == 0 && coff_v % 4 == 0 && t_max >= 0 &&
                    static_cast<int64_t>(t_max + 1) * h * w <= slots_cap,
                "bank_write_sets: slot %d does not fit capacity %lld", t_max, (long long)slots_cap);
  const int64_t total = static_cast<int64_t>(k_objects) * h * w * 160;
  launch_pdl(bank_write_kernel<true>, capped_grid(total), kThreads, 0, ST(s),
      reinterpret_cast<const float4*>(halo), k_objects, h, w, cstride / 4, coff_k / 4, coff_v / 4,
      reinterpret_cast<float4*>(bank_k), reinterpret_cast<float4*>(bank_v), slots_cap, t_max, dyn_t, k_objects / sets,
      nullptr, 0);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_bank_write_groups(const float* halo, int maps, int groups, const int32_t* first, int h,
                                                 int w, int cstride, int coff_k, int coff_v, float* bank_k,
                                                 float* bank_v, int64_t slots_cap, int t_max, const int32_t* dyn_t,
                                                 mivos_stream_t s) {
  MIVOS_REQUIRE(dyn_t, "bank_write_groups: null frame array (one device-side bank frame per group)");
  MIVOS_REQUIRE(first, "bank_write_groups: null group table (groups + 1 device-side first maps)");
  MIVOS_REQUIRE(groups >= 1 && groups <= maps, "bank_write_groups: %d groups for %d maps (1 <= groups <= maps)", groups,
                maps);
  MIVOS_REQUIRE(halo && bank_k && bank_v && AL16(halo) && AL16(bank_k) && AL16(bank_v),
                "bank_write_groups: null/unaligned pointer");
  MIVOS_REQUIRE(cstride % 4 == 0 && coff_k % 4 == 0 && coff_v % 4 == 0 && t_max >= 0 &&
                    static_cast<int64_t>(t_max + 1) * h * w <= slots_cap,
                "bank_write_groups: slot %d does not fit capacity %lld", t_max, (long long)slots_cap);
  const int64_t total = static_cast<int64_t>(maps) * h * w * 160;
  launch_pdl(bank_write_kernel<true, true>, capped_grid(total), kThreads, 0, ST(s),
      reinterpret_cast<const float4*>(halo), maps, h, w, cstride / 4, coff_k / 4, coff_v / 4,
      reinterpret_cast<float4*>(bank_k), reinterpret_cast<float4*>(bank_v), slots_cap, t_max, dyn_t, 0, first, groups);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_bank_from_nchw(const float* keys, const float* values, int k_objects,
                                              int t, int hw, float* bank_k, float* bank_v,
                                              int64_t slots_cap, mivos_stream_t s) {
  MIVOS_REQUIRE(keys && values && bank_k && bank_v, "bank_from_nchw: null pointer");
  const int64_t slots = static_cast<int64_t>(t) * hw;
  MIVOS_REQUIRE(slots <= slots_cap && slots > 0, "bank_from_nchw: %lld slots exceed capacity %lld",
                (long long)slots, (long long)slots_cap);
  dim3 gk(static_cast<unsigned>(ceil_div64(slots, 32)), 4, k_objects);
  launch_pdl(bank_transpose_kernel, gk, 256, 0, ST(s), keys, 128, slots, bank_k, slots_cap);
  MIVOS_LAUNCHED();
  dim3 gv(static_cast<unsigned>(ceil_div64(slots, 32)), 16, k_objects);
  launch_pdl(bank_transpose_kernel, gv, 256, 0, ST(s), values, 512, slots, bank_v, slots_cap);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_upsample4x_sigmoid_aggregate(const float* logits, int k_objects, int h4,
                                                            int w4, int cstride, int coff,
                                                            float* raw_out, float* prob_out, int groups,
                                                            mivos_stream_t s) {
  MIVOS_REQUIRE(logits && (raw_out || prob_out), "upsample4x: null pointer");
  MIVOS_REQUIRE(k_objects >= 1 && k_objects <= kMaxObjects, "upsample4x: %d objects (max %d)", k_objects, kMaxObjects);
  MIVOS_REQUIRE(groups >= 1, "upsample4x: groups must be >= 1");
  const int64_t plane = 16ll * h4 * w4;
  launch_pdl(upsample4x_sigmoid_aggregate_kernel<false>, capped_grid(plane * groups), kThreads, 0, ST(s), 
      logits, k_objects, h4, w4, cstride, coff, raw_out, prob_out, groups, nullptr);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_upsample4x_sigmoid_aggregate_groups(const float* logits, int maps, int groups,
                                                                   const int32_t* first, int h4, int w4, int cstride,
                                                                   int coff, float* raw_out, float* prob_out,
                                                                   mivos_stream_t s) {
  MIVOS_REQUIRE(first, "upsample4x_groups: null group table (groups + 1 device-side first maps)");
  MIVOS_REQUIRE(logits && (raw_out || prob_out), "upsample4x_groups: null pointer");
  MIVOS_REQUIRE(groups >= 1 && groups <= maps, "upsample4x_groups: %d groups for %d maps (1 <= groups <= maps)", groups,
                maps);
  MIVOS_REQUIRE(maps <= kMaxObjects * groups, "upsample4x_groups: %d maps in %d groups (max %d objects per group)", maps,
                groups, kMaxObjects);
  MIVOS_REQUIRE(h4 >= 1 && w4 >= 1 && coff >= 0 && coff < cstride, "upsample4x_groups: bad shape");
  const int64_t plane = 16ll * h4 * w4;
  launch_pdl(upsample4x_sigmoid_aggregate_kernel<true>, capped_grid(plane * groups), kThreads, 0, ST(s), logits, maps,
             h4, w4, cstride, coff, raw_out, prob_out, groups, first);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_halo_upsample_to_plane(const float* halo, int n, int hs, int ws, int cstride, int coff,
                                                      int out_h, int out_w, int apply_sigmoid, float* out,
                                                      mivos_stream_t s) {
  MIVOS_REQUIRE(halo && out && n > 0 && hs > 0 && ws > 0 && out_h > 0 && out_w > 0 && coff >= 0 && coff < cstride,
                "halo_upsample_to_plane: bad arguments");
  const float sy = static_cast<float>(hs) / static_cast<float>(out_h), sx = static_cast<float>(ws) / static_cast<float>(out_w);
  const int64_t total = static_cast<int64_t>(n) * out_h * out_w;
  launch_pdl(halo_upsample_to_plane_kernel, capped_grid(total), kThreads, 0, ST(s), halo, n, hs, ws, cstride, coff, out_h,
             out_w, sy, sx, apply_sigmoid, out);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_overlay_davis(const uint8_t* image_hwc, const uint8_t* mask, int t, int h, int w,
                                             const uint8_t* colors, int ncolors, double alpha, int fade, uint8_t* out,
                                             mivos_stream_t s) {
  MIVOS_REQUIRE(image_hwc && mask && colors && out && t > 0 && h > 0 && w > 0 && ncolors > 0 && ncolors <= 256,
                "overlay_davis: bad arguments");
  MIVOS_REQUIRE(alpha >= 0.0 && alpha <= 1.0, "overlay_davis: alpha %f outside [0,1]", alpha);
  const int64_t total = static_cast<int64_t>(t) * h * w;
  launch_pdl(overlay_davis_kernel, capped_grid(total), kThreads, 0, ST(s), image_hwc, mask, t, h, w, colors, ncolors, alpha,
             fade, out);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_aggregate_wbg(const float* prob, int k_objects, int64_t hw, int keep_bg,
                                             int hard, float* out, mivos_stream_t s) {
  MIVOS_REQUIRE(prob && out, "aggregate_wbg: null pointer");
  MIVOS_REQUIRE(k_objects >= 1 && k_objects <= kMaxObjects, "aggregate_wbg: %d objects (max %d)", k_objects, kMaxObjects);
  launch_pdl(aggregate_wbg_kernel, capped_grid(hw), kThreads, 0, ST(s), prob, k_objects, hw, keep_bg, hard, out);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_upsample4x_sigmoid_aggregate_planes(const float* logits, int k_objects, int h4, int w4,
                                                                   int cstride, int coff, float* raw_out,
                                                                   float* prob_out, int groups, mivos_stream_t s) {
  MIVOS_REQUIRE(logits && (raw_out || prob_out), "upsample4x_planes: null pointer");
  MIVOS_REQUIRE(k_objects >= 1 && k_objects <= MIVOS_MAX_OBJECTS, "upsample4x_planes: %d objects (1 to %d)", k_objects,
                MIVOS_MAX_OBJECTS);
  MIVOS_REQUIRE(groups >= 1 && h4 >= 1 && w4 >= 1 && coff >= 0 && coff < cstride, "upsample4x_planes: bad shape");
  const int64_t plane = 16ll * h4 * w4;
  const int64_t pgs = (k_objects + 1) * plane;  // prob volume of one group
  launch_pdl(upsample4x_sigmoid_planes_kernel, capped_grid(plane * k_objects * groups), kThreads, 0, ST(s), logits,
             k_objects, h4, w4, cstride, coff, groups, raw_out, prob_out ? prob_out + plane : nullptr, pgs);
  MIVOS_LAUNCHED();
  if (prob_out) {  // in place: the object planes written above become the result
    launch_pdl(aggregate_planes_kernel, capped_grid(plane * groups), kThreads, 0, ST(s),
               static_cast<const float*>(prob_out + plane), k_objects, plane, groups, pgs, prob_out, pgs, 1, 0);
    MIVOS_LAUNCHED();
  }
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_aggregate_wbg_planes(const float* prob, int k_objects, int64_t hw, int keep_bg, int hard,
                                                    float* out, mivos_stream_t s) {
  MIVOS_REQUIRE(prob && out, "aggregate_wbg_planes: null pointer");
  MIVOS_REQUIRE(k_objects >= 1 && k_objects <= MIVOS_MAX_OBJECTS, "aggregate_wbg_planes: %d objects (1 to %d)",
                k_objects, MIVOS_MAX_OBJECTS);
  MIVOS_REQUIRE(hw >= 1 && hard >= 0 && hard <= 3, "aggregate_wbg_planes: bad arguments");
  launch_pdl(aggregate_planes_kernel, capped_grid(hw), kThreads, 0, ST(s), prob, k_objects, hw, 1, int64_t{0}, out,
             int64_t{0}, keep_bg ? 1 : 0, hard);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_argmax_unpad(const float* prob, int k_plus_1, int t, int nh, int nw,
                                            int pad_l, int pad_t, int h, int w, uint8_t* masks_padded,
                                            uint8_t* masks_out, mivos_stream_t s) {
  MIVOS_REQUIRE(prob && masks_padded && k_plus_1 >= 1 && k_plus_1 <= MIVOS_MAX_OBJECTS + 1, "argmax_unpad: bad arguments");
  const int64_t total = static_cast<int64_t>(t) * nh * nw;
  launch_pdl(argmax_unpad_kernel, capped_grid(total), kThreads, 0, ST(s), prob, k_plus_1, t, nh, nw, pad_l, pad_t,
                                                                  h, w, masks_padded, masks_out);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_pad2d(const float* in, int planes, int h, int w, int pad_l, int pad_r,
                                     int pad_t, int pad_b, float* out, mivos_stream_t s) {
  MIVOS_REQUIRE(in && out && pad_l >= 0 && pad_r >= 0 && pad_t >= 0 && pad_b >= 0, "pad2d: bad arguments");
  const int nh = h + pad_t + pad_b, nw = w + pad_l + pad_r;
  const int64_t total = static_cast<int64_t>(planes) * nh * nw;
  launch_pdl(pad2d_kernel, capped_grid(total), kThreads, 0, ST(s), in, planes, h, w, pad_l, pad_t, nh, nw, out);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_halo_sigmoid_to_plane(const float* halo, int h, int w, int cstride,
                                                     int coff, float* plane, mivos_stream_t s) {
  MIVOS_REQUIRE(halo && plane, "halo_sigmoid_to_plane: null pointer");
  launch_pdl(halo_sigmoid_to_plane_kernel, capped_grid(static_cast<int64_t>(h) * w), kThreads, 0, ST(s), 
      halo, h, w, cstride, coff, plane);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_halo_to_pixels(const float* halo, int n, int h, int w, int cstride, int coff,
                                              int c, float* out, mivos_stream_t s) {
  MIVOS_REQUIRE(halo && out && AL16(halo) && AL16(out) && c % 4 == 0 && cstride % 4 == 0 && coff % 4 == 0 &&
                    coff + c <= cstride,
                "halo_to_pixels: bad arguments");
  const int64_t total = static_cast<int64_t>(n) * h * w * (c / 4);
  launch_pdl(halo_to_pixels_kernel, capped_grid(total), kThreads, 0, ST(s), 
      reinterpret_cast<const float4*>(halo), n, h, w, cstride / 4, coff / 4, c / 4, reinterpret_cast<float4*>(out));
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_frames_u8_normalize(const uint8_t* frames_hwc, int t, int h, int w, float* out,
                                                   mivos_stream_t s) {
  MIVOS_REQUIRE(frames_hwc && out && t > 0 && h > 0 && w > 0, "frames_u8_normalize: bad arguments");
  const int64_t ppf = static_cast<int64_t>(h) * w, total = ppf * t;
  launch_pdl(frames_u8_normalize_kernel, capped_grid(total), kThreads, 0, ST(s), frames_hwc, ppf, total, out);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_store_words(int64_t* dst64, int n64, const int64_t* vals64, int32_t* dst32, int n32,
                                           int v0, int v1, int v2, int v3, mivos_stream_t s) {
  MIVOS_REQUIRE(n64 >= 0 && n64 <= 64 && n32 >= 0 && n32 <= 4 && (n64 == 0 || (dst64 && vals64)) && (n32 == 0 || dst32),
                "store_words: bad arguments");
  StoreWords w;
  for (int i = 0; i < 64; ++i) w.v[i] = i < n64 ? vals64[i] : 0;
  launch_pdl(store_words_kernel, 1, 64, 0, ST(s), dst64, n64, w, dst32, n32, v0, v1, v2, v3);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_copy_segments(const int64_t* fixed, const int64_t* dyn, const int64_t* bytes, int n,
                                             int dyn_is_src, int64_t max_bytes, mivos_stream_t s) {
  MIVOS_REQUIRE(fixed && dyn && bytes && n >= 1 && n <= 65535 && max_bytes >= 16, "copy_segments: bad arguments");
  const dim3 grid(capped_grid(max_bytes / 16), n);
  launch_pdl(copy_segments_kernel, grid, kThreads, 0, ST(s), fixed, dyn, bytes, dyn_is_src);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_deliver_planes(const float* planes, const int64_t* table, int clips, int nh, int nw,
                                              mivos_stream_t s) {
  MIVOS_REQUIRE(planes && table && AL16(planes) && clips >= 1 && clips <= 65535 && nh >= 1 && nw >= 1 &&
                    (static_cast<int64_t>(nh) * nw) % kDeliverPix == 0,
                "deliver_planes: bad arguments (clips %d, %dx%d)", clips, nh, nw);
  const int64_t spans = (static_cast<int64_t>(nh) * nw + kDeliverSpan - 1) / kDeliverSpan;
  const dim3 grid(static_cast<unsigned>(spans < num_sms() * 4 ? spans : num_sms() * 4), clips);
  launch_pdl(deliver_planes_kernel, grid, kThreads, 0, ST(s), planes, table, nh, nw);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_store_i32(int32_t* dst, int n, int v0, int v1, int v2, int v3, mivos_stream_t s) {
  MIVOS_REQUIRE(dst && n >= 1 && n <= 4, "store_i32: bad arguments");
  launch_pdl(store_i32_kernel, 1, 32, 0, ST(s), dst, n, v0, v1, v2, v3);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}
