// HALO-map kernels that exist in two element types: fp32 (TF32 tensor-core path) and fp16 (the
// precision the reference GUI runs in under torch.cuda.amp.autocast, interactive_gui.py:990).
// All are HBM-bound streaming kernels working on 16-byte vectors (4 x fp32 / 8 x fp16) with the
// channel index fastest, so every warp access is a run of full 128-byte lines; arithmetic is done
// in fp32 and rounded to nearest-even on store.
#include "host_util.h"
#include "pdl.cuh"

#include <atomic>
#include <cuda_fp16.h>

namespace mivos {
extern std::atomic<int64_t> g_launches;
namespace {

constexpr int kThreads = 256;

#define MIVOS_LAUNCHED()                                \
  do {                                                  \
    g_launches.fetch_add(1, std::memory_order_relaxed); \
    MIVOS_CUDA_OK(cudaGetLastError());                  \
  } while (0)

inline unsigned capped_grid(int64_t work) {
  const int64_t cap = num_sms() * 16ll;
  int64_t g = (work + kThreads - 1) / kThreads;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<unsigned>(g);
}

// 16-byte vector of T viewed as floats
template <typename T>
struct V16;
template <>
struct V16<float> {
  static constexpr int N = 4;
  __device__ static void load(const void* p, float (&f)[4]) {
    const float4 v = *reinterpret_cast<const float4*>(p);
    f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  }
  __device__ static void store(void* p, const float (&f)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  }
};
template <>
struct V16<__half> {
  static constexpr int N = 8;
  __device__ static void load(const void* p, float (&f)[8]) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
      f[2 * i] = t.x;
      f[2 * i + 1] = t.y;
    }
  }
  __device__ static void store(void* p, const float (&f)[8]) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<const uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
  }
};

template <typename T>
__device__ __forceinline__ T from_float(float v);
template <>
__device__ __forceinline__ float from_float<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half from_float<__half>(float v) { return __float2half_rn(v); }
__device__ __forceinline__ float to_float(float v) { return v; }
__device__ __forceinline__ float to_float(__half v) { return __half2float(v); }

// ------------------------------------------------------------------------------------------
// stem gather: 7x7 / stride 2 / pad 3 windows of cat(frame, mask, others) -> im2col matrix
// [K*(H/2+2)*(W/2+2), kpad], k = (ky*7 + kx)*CIN + c.
// One CTA per output row (halo rows included: they are written as zeros).  Phase 1 stages the 7
// input rows the output row needs into shared memory, channel-interleaved [ky][x + 3][c] in the
// output element type, with the 3-pixel zero padding materialised; the "others" channel (sum of
// the other objects' masks, in object order — prop_net.py:150-157) is formed here.  In that layout
// the 7 x CIN values of a window row are CONTIGUOUS, so phase 2 is 7 short copies per output pixel:
// a warp writes one 512-byte (fp16, kpad 256) matrix row with one 16-byte store per lane.  Global
// reads are coalesced along x, every input row is read by the ~3.5 CTAs that need it (L2 hits).
// (The first version computed (ky, kx, c) per element and issued one scalar global load per
// element: 88 us for the 54 MB matrix; this one is bounded by the matrix write.)
constexpr int kStemThreads = 512;
template <int CIN, typename T>
__global__ void __launch_bounds__(kStemThreads)
stem_gather_kernel(const float* __restrict__ frame, const float* __restrict__ masks, int kobj, int h, int w,
                   T* __restrict__ out, int kpad, int64_t frame_gstride, int64_t mask_gstride) {
  mivos::pdl_prologue();
  extern __shared__ __align__(16) uint8_t stem_smem[];
  T* win = reinterpret_cast<T*>(stem_smem);  // [7][w + 6][CIN]
  const int ho = h / 2, wo = w / 2;
  const int wp = wo + 2;
  const int yo = static_cast<int>(blockIdx.x) - 1;  // output row, -1 and ho are halo rows
  const int img = blockIdx.y;                       // output image: group (clip) major
  // CIN == 5: image = object `obj` of group `img / kobj` (own frame, own K masks); otherwise a batch of frames
  const int obj = CIN == 5 ? img % kobj : img;
  if constexpr (CIN == 5) {
    frame += static_cast<int64_t>(img / kobj) * frame_gstride;
    masks += static_cast<int64_t>(img / kobj) * mask_gstride;
  }
  const int64_t plane = static_cast<int64_t>(h) * w;
  const int rowlen = (w + 6) * CIN;
  const bool live_row = yo >= 0 && yo < ho;

  if (live_row) {
    // ---- phase 1: 7 rows x (w + 6) pixels x CIN channels
    // CIN == 5: one frame + K masks (memorize); otherwise `frame` is a batch of CIN-channel images
    constexpr int NF = CIN == 5 ? 3 : CIN;
    const float* fr = frame + (CIN == 5 ? 0 : static_cast<int64_t>(obj) * CIN * plane);
    // (latency-bound: ~12 staged pixels per thread, 3-5 independent global loads each)
#pragma unroll 4
    for (int i = threadIdx.x; i < 7 * (w + 6); i += kStemThreads) {
      const int ky = i / (w + 6), xs = i - ky * (w + 6);
      const int y = 2 * yo + ky - 3, x = xs - 3;
      float v[CIN];
#pragma unroll
      for (int c = 0; c < CIN; ++c) v[c] = 0.f;
      if (y >= 0 && y < h && x >= 0 && x < w) {
        const int64_t pix = static_cast<int64_t>(y) * w + x;
#pragma unroll
        for (int c = 0; c < NF; ++c) v[c] = fr[c * plane + pix];
        if constexpr (CIN == 5) {
          float own = 0.f, others = 0.f;
          for (int j = 0; j < kobj; ++j) {
            const float m = masks[j * plane + pix];
            if (j == obj) own = m;
            else others += m;
          }
          v[3] = own;
          v[CIN - 1] = others;
        }
      }
#pragma unroll
      for (int c = 0; c < CIN; ++c) win[(ky * (w + 6) + xs) * CIN + c] = from_float<T>(v[c]);
    }
  }
  __syncthreads();

  // ---- phase 2: one warp per output pixel (halo pixels -> zeros), V elements per lane per store
  constexpr int V = 16 / static_cast<int>(sizeof(T));
  constexpr int RUN = 7 * CIN;  // contiguous elements of one window row
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int64_t row_base = (static_cast<int64_t>(img) * (ho + 2) + yo + 1) * wp;
  for (int xp = warp; xp < wp; xp += nwarps) {
    const int xo = xp - 1;
    const bool live = live_row && xo >= 0 && xo < wo;
    T* orow = out + (row_base + xp) * kpad;
    const T* src = win + 2 * xo * CIN;  // window starts at input x = 2 xo - 3, i.e. staged x = 2 xo
    for (int k0 = lane * V; k0 < kpad; k0 += 32 * V) {
      alignas(16) T vals[V];
#pragma unroll
      for (int e = 0; e < V; ++e) {
        const int k = k0 + e;
        const int ky = k / RUN, r = k - ky * RUN;
        vals[e] = (live && k < 7 * RUN) ? src[ky * rowlen + r] : from_float<T>(0.f);
      }
      *reinterpret_cast<uint4*>(orow + k0) = *reinterpret_cast<const uint4*>(vals);
    }
  }
}

// ------------------------------------------------------------------------------------------
// space-to-depth stem gather (mivos_stem_gather_s2d): for every HALO row (Y, X) of the half-resolution
// output map, the 2 input rows x 8 input pixels x CIN channels its four horizontal taps read,
//   out[row, py*8*CIN + j*CIN + c] = in[c, 2Y+py, 2X-4+j]   (zero outside the image).
// One CTA per output row: the two input rows are staged channel-interleaved [py][x + 4][c] in the output
// element type with 4 pixels of zero padding on each side (the "others" channel of the memorize stem is
// formed here), so a matrix row is two contiguous runs of 8*CIN staged values; a thread assembles one
// 16-byte piece, a warp writes 512 contiguous bytes.
template <int CIN, typename T>
__global__ void __launch_bounds__(256)
stem_s2d_gather_kernel(const float* __restrict__ frame, const float* __restrict__ masks, int kobj, int h, int w,
                       T* __restrict__ out, int kpad, int64_t frame_gstride, int64_t mask_gstride) {
  mivos::pdl_prologue();
  extern __shared__ __align__(16) uint8_t s2d_smem[];
  T* rowbuf = reinterpret_cast<T*>(s2d_smem);  // [2][w + 8][CIN]
  const int ho = h / 2, wo = w / 2;
  const int wp = wo + 2;
  const int yo = static_cast<int>(blockIdx.x) - 1;  // output row; -1 and ho are border rows (zeros)
  const int img = blockIdx.y;
  const int obj = CIN == 5 ? img % kobj : img;
  if constexpr (CIN == 5) {
    frame += static_cast<int64_t>(img / kobj) * frame_gstride;
    masks += static_cast<int64_t>(img / kobj) * mask_gstride;
  }
  const int64_t plane = static_cast<int64_t>(h) * w;
  const int rowlen = (w + 8) * CIN;
  const bool live_row = yo >= 0 && yo < ho;
  if (live_row) {
    constexpr int NF = CIN == 5 ? 3 : CIN;
    const float* fr = frame + (CIN == 5 ? 0 : static_cast<int64_t>(obj) * CIN * plane);
    for (int i = threadIdx.x; i < 2 * (w + 8); i += blockDim.x) {
      const int py = i / (w + 8), xs = i - py * (w + 8);
      const int y = 2 * yo + py, x = xs - 4;
      float v[CIN];
#pragma unroll
      for (int c = 0; c < CIN; ++c) v[c] = 0.f;
      if (x >= 0 && x < w) {
        const int64_t pix = static_cast<int64_t>(y) * w + x;
#pragma unroll
        for (int c = 0; c < NF; ++c) v[c] = fr[c * plane + pix];
        if constexpr (CIN == 5) {
          float own = 0.f, others = 0.f;
          for (int j = 0; j < kobj; ++j) {
            const float m = masks[j * plane + pix];
            if (j == obj) own = m;
            else others += m;
          }
          v[3] = own;
          v[4] = others;
        }
      }
#pragma unroll
      for (int c = 0; c < CIN; ++c) rowbuf[(py * (w + 8) + xs) * CIN + c] = from_float<T>(v[c]);
    }
  }
  __syncthreads();
  constexpr int V = 16 / static_cast<int>(sizeof(T));  // elements per 16-byte piece
  constexpr int RUN = 8 * CIN;                          // staged values per input row of a matrix row
  static_assert(RUN % V == 0, "a 16-byte piece must not straddle the two input rows");
  const int pieces = kpad / V;
  const int64_t row_base = (static_cast<int64_t>(img) * (ho + 2) + yo + 1) * wp;
  for (int i = threadIdx.x; i < wp * pieces; i += blockDim.x) {
    const int xp = i / pieces, pc = i - xp * pieces;
    const int xo = xp - 1;
    const bool live = live_row && xo >= 0 && xo < wo;
    const int k0 = pc * V;
    alignas(16) T vals[V];
#pragma unroll
    for (int e = 0; e < V; ++e) vals[e] = from_float<T>(0.f);
    if (live && k0 < 2 * RUN) {
      const int py = k0 / RUN, j0 = k0 - py * RUN;
      const T* src = rowbuf + py * rowlen + 2 * xo * CIN + j0;  // staged x = 2 xo - 4 + 4
#pragma unroll
      for (int e = 0; e < V; ++e) vals[e] = src[e];
    }
    *reinterpret_cast<uint4*>(out + (row_base + xp) * kpad + k0) = *reinterpret_cast<const uint4*>(vals);
  }
}

// ------------------------------------------------------------------------------------------
// stride-2 gather from a HALO map into an im2col matrix (rows = HALO rows of the output map);
// pure 16-byte copies, so one kernel serves both element types (cv = channels / vector width).
__global__ void gather_s2_kernel(const uint4* __restrict__ in, int n, int h, int w, int cv,
                                 int in_cstride_v, int ks, uint4* __restrict__ out, int out_cstride_v) {
  mivos::pdl_prologue();
  const int ho = h / 2, wo = w / 2;
  const int wpo = wo + 2, wpi = w + 2;
  const int kk = ks * ks;
  const int64_t rows = static_cast<int64_t>(n) * (ho + 2) * wpo;
  const int64_t total = rows * kk * cv;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % cv);
    const int64_t t1 = i / cv;
    const int tap = static_cast<int>(t1 % kk);
    const int64_t r = t1 / kk;
    const int64_t per_img = static_cast<int64_t>(ho + 2) * wpo;
    const int img = static_cast<int>(r / per_img);
    const int rem = static_cast<int>(r - img * per_img);
    const int yo = rem / wpo - 1, xo = rem % wpo - 1;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (yo >= 0 && yo < ho && xo >= 0 && xo < wo) {
      const int ky = tap / ks, kx = tap - ky * ks;
      // input pixel (2*yo + ky - ks/2, 2*xo + kx - ks/2); +1 for the halo offset
      const int yi = 2 * yo + ky - ks / 2 + 1, xi = 2 * xo + kx - ks / 2 + 1;
      const int64_t rin = (static_cast<int64_t>(img) * (h + 2) + yi) * wpi + xi;
      v = in[rin * in_cstride_v + ci];
    }
    out[r * out_cstride_v + tap * cv + ci] = v;
  }
}

// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void maxpool3x3s2_kernel(const T* __restrict__ in, int n, int h, int w, int cv, T* __restrict__ out) {
  mivos::pdl_prologue();
  constexpr int N = V16<T>::N;
  const int ho = h / 2, wo = w / 2;
  const int wpo = wo + 2, wpi = w + 2;
  const int64_t total = static_cast<int64_t>(n) * ho * wo * cv;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % cv);
    int64_t t1 = i / cv;
    const int xo = static_cast<int>(t1 % wo);
    t1 /= wo;
    const int yo = static_cast<int>(t1 % ho);
    const int img = static_cast<int>(t1 / ho);
    // inputs are post-ReLU (>= 0), so the zero halo is equivalent to the -inf pad of MaxPool2d
    float m[N];
#pragma unroll
    for (int e = 0; e < N; ++e) m[e] = 0.f;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int yi = 2 * yo + ky, xi = 2 * xo + kx;  // halo coords of (2yo+ky-1, 2xo+kx-1)
        float v[N];
        V16<T>::load(in + (((static_cast<int64_t>(img) * (h + 2) + yi) * wpi + xi) * cv + ci) * N, v);
#pragma unroll
        for (int e = 0; e < N; ++e) m[e] = fmaxf(m[e], v[e]);
      }
    V16<T>::store(out + (((static_cast<int64_t>(img) * (ho + 2) + yo + 1) * wpo + xo + 1) * cv + ci) * N, m);
  }
}

// ------------------------------------------------------------------------------------------
// bilinear source index, align_corners=False (ATen area_pixel_compute_source_index)
__device__ __forceinline__ void bilin(int dst, float scale, int in_size, int& i0, int& i1, float& l1) {
  float src = scale * (static_cast<float>(dst) + 0.5f) - 0.5f;
  if (src < 0.f) src = 0.f;
  i0 = static_cast<int>(src);
  i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
  l1 = src - static_cast<float>(i0);
}

template <typename T>
__global__ void upsample2x_add_kernel(T* __restrict__ x, const T* __restrict__ up, int n, int h, int w, int cv,
                                      T* __restrict__ x_relu, const T* __restrict__ skip, int per_skip) {
  mivos::pdl_prologue();
  constexpr int N = V16<T>::N;
  const int hs = h / 2, ws = w / 2;
  const int64_t total = static_cast<int64_t>(n) * h * w * cv;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % cv);
    int64_t t1 = i / cv;
    const int xo = static_cast<int>(t1 % w);
    t1 /= w;
    const int yo = static_cast<int>(t1 % h);
    const int img = static_cast<int>(t1 / h);
    int y0, y1, x0, x1;
    float ly, lx;
    bilin(yo, 0.5f, hs, y0, y1, ly);
    bilin(xo, 0.5f, ws, x0, x1, lx);
    const float hy = 1.f - ly, hx = 1.f - lx;
    const int64_t base = static_cast<int64_t>(img) * (hs + 2);
    float v00[N], v01[N], v10[N], v11[N], xv[N];
    V16<T>::load(up + (((base + y0 + 1) * (ws + 2) + x0 + 1) * cv + ci) * N, v00);
    V16<T>::load(up + (((base + y0 + 1) * (ws + 2) + x1 + 1) * cv + ci) * N, v01);
    V16<T>::load(up + (((base + y1 + 1) * (ws + 2) + x0 + 1) * cv + ci) * N, v10);
    V16<T>::load(up + (((base + y1 + 1) * (ws + 2) + x1 + 1) * cv + ci) * N, v11);
    const int64_t o = (((static_cast<int64_t>(img) * (h + 2) + yo + 1) * (w + 2) + xo + 1) * cv + ci) * N;
    // `skip` (one map per `per_skip` consecutive images: a frame's skip path broadcast over its objects)
    // replaces x as the addend: x = skip + up2x(up)
    if (skip) V16<T>::load(skip + (((static_cast<int64_t>(img / per_skip) * (h + 2) + yo + 1) * (w + 2) + xo + 1) * cv + ci) * N, xv);
    else V16<T>::load(x + o, xv);
    float r[N];
#pragma unroll
    for (int e = 0; e < N; ++e) xv[e] += hy * (hx * v00[e] + lx * v01[e]) + ly * (hx * v10[e] + lx * v11[e]);
    V16<T>::store(x + o, xv);
    if (x_relu) {
#pragma unroll
      for (int e = 0; e < N; ++e) r[e] = fmaxf(xv[e], 0.f);
      V16<T>::store(x_relu + o, r);
    }
  }
}

// ------------------------------------------------------------------------------------------
// channel-window copy between HALO maps with optional ReLU and type conversion; 4 channels/thread
template <typename TS, typename TD>
__global__ void halo_copy_kernel(const TS* __restrict__ src, int src_n, int src_cs, int src_co, TD* __restrict__ dst,
                                 int dst_cs, int dst_co, int n, int h, int w, int c4, int relu) {
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
    const int simg = img / (n / src_n);  // src_n maps broadcast over n / src_n consecutive images each
    const int64_t rs = (static_cast<int64_t>(simg) * (h + 2) + y + 1) * (w + 2) + x + 1;
    const int64_t rd = (static_cast<int64_t>(img) * (h + 2) + y + 1) * (w + 2) + x + 1;
    const TS* s = src + rs * src_cs + src_co + ci * 4;
    TD* d = dst + rd * dst_cs + dst_co + ci * 4;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float v = to_float(s[e]);
      if (relu) v = fmaxf(v, 0.f);
      d[e] = from_float<TD>(v);
    }
  }
}

// ------------------------------------------------------------------------------------------
// [channels x pixels] <-> [pixels x channels] transposes through a padded 32x32 smem tile.
// grid: (pixel tiles, channel tiles, planes).  NCHW side is always fp32 (the reference's layout).
template <typename T>
__global__ void halo_to_nchw_kernel(const T* __restrict__ halo, int h, int w, int cstride, int coff, int c,
                                    float* __restrict__ nchw) {
  mivos::pdl_prologue();
  __shared__ float tile[32][33];
  const int img = blockIdx.z;
  const int hw = h * w;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int p = p0 + j, ch = c0 + tx;
    float v = 0.f;
    if (p < hw && ch < c) {
      const int y = p / w, x = p - y * w;
      v = to_float(halo[((static_cast<int64_t>(img) * (h + 2) + y + 1) * (w + 2) + x + 1) * cstride + coff + ch]);
    }
    tile[j][tx] = v;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int ch = c0 + j, p = p0 + tx;
    if (p < hw && ch < c) nchw[(static_cast<int64_t>(img) * c + ch) * hw + p] = tile[tx][j];
  }
}

template <typename T>
__global__ void nchw_to_halo_kernel(const float* __restrict__ nchw, int h, int w, int c, T* __restrict__ halo,
                                    int cstride, int coff, int relu) {
  mivos::pdl_prologue();
  __shared__ float tile[32][33];
  const int img = blockIdx.z;
  const int hw = h * w;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int j = ty; j < 32; j += 8) {
    const int ch = c0 + j, p = p0 + tx;
    float v = 0.f;
    if (p < hw && ch < c) v = nchw[(static_cast<int64_t>(img) * c + ch) * hw + p];
    tile[j][tx] = relu ? fmaxf(v, 0.f) : v;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int p = p0 + j, ch = c0 + tx;
    if (p < hw && ch < c) {
      const int y = p / w, x = p - y * w;
      halo[((static_cast<int64_t>(img) * (h + 2) + y + 1) * (w + 2) + x + 1) * cstride + coff + ch] =
          from_float<T>(tile[tx][j]);
    }
  }
}

// FusionNet input (fusion_net.py:35-40): cat(im, seg1, seg2, attn, time) -> HALO (1,H,W,cpad),
// channels 9..cpad-1 zero
template <typename T>
__global__ void fusion_gather_kernel(const float* __restrict__ im, const float* __restrict__ seg1,
                                     const float* __restrict__ seg2, const float* __restrict__ attn, float nc,
                                     float nr, int h, int w, T* __restrict__ out, int cpad) {
  mivos::pdl_prologue();
  const int64_t plane = static_cast<int64_t>(h) * w;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < plane;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / w), x = static_cast<int>(i - static_cast<int64_t>(y) * w);
    T* o = out + (static_cast<int64_t>(y + 1) * (w + 2) + x + 1) * cpad;
    const float v[9] = {im[i], im[plane + i], im[2 * plane + i], seg1[i], seg2[i], attn[i], attn[plane + i], nc, nr};
#pragma unroll
    for (int c = 0; c < 9; ++c) o[c] = from_float<T>(v[c]);
    for (int c = 9; c < cpad; ++c) o[c] = from_float<T>(0.f);
  }
}


// ------------------------------------------------------------------------------------------
// dilated 3x3 / stride 1 / pad = dilation gather from a HALO map into an im2col matrix whose rows
// are the HALO rows of the (same-size) output map: out[r, tap*c + ci] = in(y + (ky-1)*d, x + (kx-1)*d)
// or 0 outside the image (s2m_resnet.py:19-20 conv3x3 with dilation, _deeplab.py:121-123 ASPPConv).
// Pure 16-byte copies (one kernel for both element types), like gather_s2_kernel.
__global__ void gather_dilated_kernel(const uint4* __restrict__ in, int n, int h, int w, int cv, int in_cstride_v,
                                      int dil, uint4* __restrict__ out, int out_cstride_v) {
  mivos::pdl_prologue();
  const int wp = w + 2;
  const int64_t per_img = static_cast<int64_t>(h + 2) * wp;
  const int64_t rows = static_cast<int64_t>(n) * per_img;
  const int64_t total = rows * 9 * cv;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % cv);
    const int64_t t1 = i / cv;
    const int tap = static_cast<int>(t1 % 9);
    const int64_t r = t1 / 9;
    const int img = static_cast<int>(r / per_img);
    const int rem = static_cast<int>(r - img * per_img);
    const int yo = rem / wp - 1, xo = rem % wp - 1;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (yo >= 0 && yo < h && xo >= 0 && xo < w) {
      const int ky = tap / 3, kx = tap - ky * 3;
      const int yi = yo + (ky - 1) * dil, xi = xo + (kx - 1) * dil;
      if (yi >= 0 && yi < h && xi >= 0 && xi < w) {
        const int64_t rin = (static_cast<int64_t>(img) * (h + 2) + yi + 1) * wp + xi + 1;
        v = in[rin * in_cstride_v + ci];
      }
    }
    out[r * out_cstride_v + tap * cv + ci] = v;
  }
}

// ------------------------------------------------------------------------------------------
// global average pool of a HALO map, written back broadcast over every interior pixel of the
// output channel window: AdaptiveAvgPool2d(1) followed by the bilinear resize of the 1x1 map
// back to (h, w) (_deeplab.py:126-138, ASPPPooling) — a constant map, so the 1x1 conv + BN + ReLU
// in between commute with the broadcast and run on the full-size map afterwards.
// grid (ceil(cv / 32), n), 256 threads = 8 pixel groups x 32 channel vectors; partial sums are
// combined in a fixed order (deterministic).
template <typename T>
__global__ void __launch_bounds__(256)
halo_avgpool_broadcast_kernel(const T* __restrict__ in, int h, int w, int cv, int in_cs, int in_co,
                              T* __restrict__ out, int out_cs, int out_co) {
  mivos::pdl_prologue();
  constexpr int N = V16<T>::N;
  __shared__ float part[8][32][N];
  __shared__ float mean[32][N];
  const int img = blockIdx.y;
  const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int cvi = static_cast<int>(blockIdx.x) * 32 + lane;
  const int hw = h * w;
  const int wp = w + 2;
  float acc[N];
#pragma unroll
  for (int e = 0; e < N; ++e) acc[e] = 0.f;
  if (cvi < cv) {
#pragma unroll 4
    for (int p = grp; p < hw; p += 8) {
      const int y = p / w, x = p - y * w;
      const int64_t row = (static_cast<int64_t>(img) * (h + 2) + y + 1) * wp + x + 1;
      float v[N];
      V16<T>::load(in + row * in_cs + in_co + cvi * N, v);
#pragma unroll
      for (int e = 0; e < N; ++e) acc[e] += v[e];
    }
  }
#pragma unroll
  for (int e = 0; e < N; ++e) part[grp][lane][e] = acc[e];
  __syncthreads();
  if (grp == 0) {
    const float inv = 1.f / static_cast<float>(hw);
#pragma unroll
    for (int e = 0; e < N; ++e) {
      float s = 0.f;
#pragma unroll
      for (int g = 0; g < 8; ++g) s += part[g][lane][e];
      mean[lane][e] = s * inv;
    }
  }
  __syncthreads();
  if (cvi < cv) {
    float m[N];
#pragma unroll
    for (int e = 0; e < N; ++e) m[e] = mean[lane][e];
    for (int p = grp; p < hw; p += 8) {
      const int y = p / w, x = p - y * w;
      const int64_t row = (static_cast<int64_t>(img) * (h + 2) + y + 1) * wp + x + 1;
      V16<T>::store(out + row * out_cs + out_co + cvi * N, m);
    }
  }
}

// ------------------------------------------------------------------------------------------
// bilinear resize (align_corners=False, any size ratio) between HALO maps, into a channel window
// of the destination: F.interpolate(x, size=..., mode='bilinear') + torch.cat at _deeplab.py:50-52.
template <typename T>
__global__ void upsample_bilinear_kernel(const T* __restrict__ src, int n, int hs, int ws, int src_cs, int src_co,
                                         T* __restrict__ dst, int h, int w, int dst_cs, int dst_co, int cv,
                                         float sy, float sx) {
  mivos::pdl_prologue();
  constexpr int N = V16<T>::N;
  const int64_t total = static_cast<int64_t>(n) * h * w * cv;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % cv);
    int64_t t1 = i / cv;
    const int xo = static_cast<int>(t1 % w);
    t1 /= w;
    const int yo = static_cast<int>(t1 % h);
    const int img = static_cast<int>(t1 / h);
    int y0, y1, x0, x1;
    float ly, lx;
    bilin(yo, sy, hs, y0, y1, ly);
    bilin(xo, sx, ws, x0, x1, lx);
    const float hy = 1.f - ly, hx = 1.f - lx;
    const int64_t base = static_cast<int64_t>(img) * (hs + 2);
    const int64_t co = src_co + ci * N;
    float v00[N], v01[N], v10[N], v11[N], r[N];
    V16<T>::load(src + ((base + y0 + 1) * (ws + 2) + x0 + 1) * src_cs + co, v00);
    V16<T>::load(src + ((base + y0 + 1) * (ws + 2) + x1 + 1) * src_cs + co, v01);
    V16<T>::load(src + ((base + y1 + 1) * (ws + 2) + x0 + 1) * src_cs + co, v10);
    V16<T>::load(src + ((base + y1 + 1) * (ws + 2) + x1 + 1) * src_cs + co, v11);
#pragma unroll
    for (int e = 0; e < N; ++e) r[e] = hy * (hx * v00[e] + lx * v01[e]) + ly * (hx * v10[e] + lx * v11[e]);
    V16<T>::store(dst + ((static_cast<int64_t>(img) * (h + 2) + yo + 1) * (w + 2) + xo + 1) * dst_cs + dst_co + ci * N, r);
  }
}

}  // namespace
}  // namespace mivos

using namespace mivos;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define AL16(p) ((reinterpret_cast<uintptr_t>(p) & 15) == 0)

extern "C" MIVOS_API int mivos_stem_gather(const float* frame, const float* masks, int k_objects, int h, int w,
                                           void* out, int kpad, int out_f16, int groups, int64_t frame_gstride,
                                           int64_t mask_gstride, mivos_stream_t s) {
  MIVOS_REQUIRE(frame && out, "stem_gather: null pointer");
  MIVOS_REQUIRE(groups >= 1 && (masks || groups == 1), "stem_gather: groups need the mask form (one frame + K masks per group)");
  MIVOS_REQUIRE(h % 2 == 0 && w % 2 == 0 && h > 0 && w > 0, "stem_gather: h,w must be even");
  const int cin = masks ? 5 : 3;
  MIVOS_REQUIRE(k_objects >= 1, "stem_gather: bad object / frame count");
  MIVOS_REQUIRE(kpad >= 49 * cin && kpad % 32 == 0, "stem_gather: kpad %d too small for cin %d", kpad, cin);
  MIVOS_REQUIRE(kpad % 8 == 0 && AL16(out), "stem_gather: output rows must be 16-byte aligned");
  const dim3 grid(h / 2 + 2, k_objects * groups);
  const int smem = 7 * (w + 6) * cin * (out_f16 ? 2 : 4);
  MIVOS_REQUIRE(smem <= 227 * 1024, "stem_gather: a %d-pixel wide frame needs %d B of shared memory", w, smem);
#define STEM(CIN_, T_)                                                                                          \
  do {                                                                                                          \
    static int configured = 0;                                                                                  \
    if (smem > configured) {                                                                                    \
      MIVOS_CUDA_OK(cudaFuncSetAttribute(stem_gather_kernel<CIN_, T_>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); \
      configured = smem;                                                                                        \
    }                                                                                                           \
    launch_pdl(stem_gather_kernel<CIN_, T_>, grid, kStemThreads, smem, ST(s), frame, masks, k_objects, h, w,    \
               static_cast<T_*>(out), kpad, frame_gstride, mask_gstride);                                       \
  } while (0)
  if (out_f16) {
    if (masks) STEM(5, __half);
    else STEM(3, __half);
  } else {
    if (masks) STEM(5, float);
    else STEM(3, float);
  }
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_stem_gather_s2d(const float* frame, const float* masks, int k_objects, int h, int w,
                                               void* out, int kpad, int out_f16, int groups, int64_t frame_gstride,
                                               int64_t mask_gstride, mivos_stream_t s) {
  MIVOS_REQUIRE(frame && out, "stem_gather_s2d: null pointer");
  MIVOS_REQUIRE(groups >= 1 && (masks || groups == 1), "stem_gather_s2d: groups need the mask form (one frame + K masks per group)");
  MIVOS_REQUIRE(h % 2 == 0 && w % 2 == 0 && h > 0 && w > 0 && k_objects >= 1, "stem_gather_s2d: h,w must be even");
  const int cin = masks ? 5 : 3;
  const int v = out_f16 ? 8 : 4;
  MIVOS_REQUIRE(kpad >= 16 * cin && kpad % v == 0 && AL16(out), "stem_gather_s2d: kpad %d too small for cin %d / unaligned", kpad, cin);
  const dim3 grid(h / 2 + 2, k_objects * groups);
  const int smem = 2 * (w + 8) * cin * (out_f16 ? 2 : 4);
  MIVOS_REQUIRE(smem <= 227 * 1024, "stem_gather_s2d: a %d-pixel wide frame needs %d B of shared memory", w, smem);
#define S2D(CIN_, T_)                                                                                      \
  do {                                                                                                     \
    static int configured = 48 * 1024;                                                                     \
    if (smem > configured) {                                                                               \
      MIVOS_CUDA_OK(cudaFuncSetAttribute(stem_s2d_gather_kernel<CIN_, T_>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); \
      configured = smem;                                                                                   \
    }                                                                                                      \
    launch_pdl(stem_s2d_gather_kernel<CIN_, T_>, grid, 256, smem, ST(s), frame, masks, k_objects, h, w,    \
               static_cast<T_*>(out), kpad, frame_gstride, mask_gstride);                                  \
  } while (0)
  if (out_f16) {
    if (masks) S2D(5, __half);
    else S2D(3, __half);
  } else {
    if (masks) S2D(5, float);
    else S2D(3, float);
  }
#undef S2D
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_stem_gather_frames(const float* frames, int n, int cin, int h, int w, void* out,
                                                  int kpad, int out_f16, mivos_stream_t s) {
  MIVOS_REQUIRE(frames && out, "stem_gather_frames: null pointer");
  MIVOS_REQUIRE(cin == 3 || cin == 6, "stem_gather_frames: %d input channels (3 or 6)", cin);
  if (cin == 3) return mivos_stem_gather(frames, nullptr, n, h, w, out, kpad, out_f16, 1, 0, 0, s);
  MIVOS_REQUIRE(h % 2 == 0 && w % 2 == 0 && h > 0 && w > 0 && n >= 1, "stem_gather_frames: bad shape");
  MIVOS_REQUIRE(kpad >= 49 * cin && kpad % 32 == 0 && AL16(out), "stem_gather_frames: kpad %d too small / unaligned", kpad);
  const float* frame = frames;
  const float* masks = nullptr;
  const int k_objects = n;
  const int64_t frame_gstride = 0, mask_gstride = 0;
  const dim3 grid(h / 2 + 2, n);
  const int smem = 7 * (w + 6) * cin * (out_f16 ? 2 : 4);
  MIVOS_REQUIRE(smem <= 227 * 1024, "stem_gather_frames: a %d-pixel wide frame needs %d B of shared memory", w, smem);
  if (out_f16) STEM(6, __half);
  else STEM(6, float);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}
#undef STEM

extern "C" MIVOS_API int mivos_gather_dilated(const void* in, int n, int h, int w, int c, int in_cstride, int dilation,
                                              void* out, int out_cstride, int f16, mivos_stream_t s) {
  MIVOS_REQUIRE(in && out && AL16(in) && AL16(out), "gather_dilated: null/unaligned pointer");
  const int v = f16 ? 8 : 4;
  MIVOS_REQUIRE(dilation >= 1 && c > 0 && c % v == 0 && in_cstride % v == 0 && out_cstride % v == 0 && c <= in_cstride &&
                    out_cstride >= 9 * c && n > 0 && h > 0 && w > 0,
                "gather_dilated: bad shape (c=%d dilation=%d)", c, dilation);
  const int64_t total = static_cast<int64_t>(n) * (h + 2) * (w + 2) * 9 * (c / v);
  launch_pdl(gather_dilated_kernel, capped_grid(total), kThreads, 0, ST(s), static_cast<const uint4*>(in), n, h, w, c / v,
             in_cstride / v, dilation, static_cast<uint4*>(out), out_cstride / v);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_halo_avgpool_broadcast(const void* in, int n, int h, int w, int c, int in_cstride,
                                                      int in_coff, void* out, int out_cstride, int out_coff, int f16,
                                                      mivos_stream_t s) {
  const int v = f16 ? 8 : 4;
  MIVOS_REQUIRE(in && out && AL16(in) && AL16(out) && n > 0 && h > 0 && w > 0 && c > 0 && c % v == 0 &&
                    in_cstride % v == 0 && in_coff % v == 0 && out_cstride % v == 0 && out_coff % v == 0 &&
                    in_coff + c <= in_cstride && out_coff + c <= out_cstride,
                "halo_avgpool_broadcast: bad arguments");
  const dim3 grid(ceil_div(c / v, 32), n);
  if (f16)
    launch_pdl(halo_avgpool_broadcast_kernel<__half>, grid, 256, 0, ST(s), static_cast<const __half*>(in), h, w, c / v,
               in_cstride, in_coff, static_cast<__half*>(out), out_cstride, out_coff);
  else
    launch_pdl(halo_avgpool_broadcast_kernel<float>, grid, 256, 0, ST(s), static_cast<const float*>(in), h, w, c / v,
               in_cstride, in_coff, static_cast<float*>(out), out_cstride, out_coff);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_upsample_bilinear(const void* src, int n, int hs, int ws, int src_cstride, int src_coff,
                                                 void* dst, int h, int w, int dst_cstride, int dst_coff, int c, int f16,
                                                 mivos_stream_t s) {
  const int v = f16 ? 8 : 4;
  MIVOS_REQUIRE(src && dst && AL16(src) && AL16(dst) && n > 0 && hs > 0 && ws > 0 && h > 0 && w > 0 && c > 0 &&
                    c % v == 0 && src_cstride % v == 0 && src_coff % v == 0 && dst_cstride % v == 0 && dst_coff % v == 0 &&
                    src_coff + c <= src_cstride && dst_coff + c <= dst_cstride,
                "upsample_bilinear: bad arguments");
  // ATen area_pixel_compute_scale for align_corners=False with an explicit output size: in / out
  const float sy = static_cast<float>(hs) / static_cast<float>(h), sx = static_cast<float>(ws) / static_cast<float>(w);
  const int64_t total = static_cast<int64_t>(n) * h * w * (c / v);
  if (f16)
    launch_pdl(upsample_bilinear_kernel<__half>, capped_grid(total), kThreads, 0, ST(s), static_cast<const __half*>(src), n,
               hs, ws, src_cstride, src_coff, static_cast<__half*>(dst), h, w, dst_cstride, dst_coff, c / v, sy, sx);
  else
    launch_pdl(upsample_bilinear_kernel<float>, capped_grid(total), kThreads, 0, ST(s), static_cast<const float*>(src), n,
               hs, ws, src_cstride, src_coff, static_cast<float*>(dst), h, w, dst_cstride, dst_coff, c / v, sy, sx);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_gather_s2(const void* in, int n, int h, int w, int c, int in_cstride, int ks,
                                         void* out, int out_cstride, int f16, mivos_stream_t s) {
  MIVOS_REQUIRE(in && out && AL16(in) && AL16(out), "gather_s2: null/unaligned pointer");
  const int v = f16 ? 8 : 4;
  MIVOS_REQUIRE((ks == 1 || ks == 3) && c % v == 0 && in_cstride % v == 0 && out_cstride % v == 0 &&
                    out_cstride >= ks * ks * c && h % 2 == 0 && w % 2 == 0,
                "gather_s2: bad shape (ks=%d c=%d)", ks, c);
  const int64_t total = static_cast<int64_t>(n) * (h / 2 + 2) * (w / 2 + 2) * ks * ks * (c / v);
  launch_pdl(gather_s2_kernel, capped_grid(total), kThreads, 0, ST(s), static_cast<const uint4*>(in), n, h, w, c / v,
                                                               in_cstride / v, ks, static_cast<uint4*>(out),
                                                               out_cstride / v);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_maxpool3x3s2(const void* in, int n, int h, int w, int c, void* out, int f16,
                                            mivos_stream_t s) {
  const int v = f16 ? 8 : 4;
  MIVOS_REQUIRE(in && out && AL16(in) && AL16(out) && c % v == 0 && h % 2 == 0 && w % 2 == 0, "maxpool: bad arguments");
  const int64_t total = static_cast<int64_t>(n) * (h / 2) * (w / 2) * (c / v);
  if (f16)
    launch_pdl(maxpool3x3s2_kernel<__half>, capped_grid(total), kThreads, 0, ST(s), static_cast<const __half*>(in), n, h, w, c / v, static_cast<__half*>(out));
  else
    launch_pdl(maxpool3x3s2_kernel<float>, capped_grid(total), kThreads, 0, ST(s), static_cast<const float*>(in), n, h, w, c / v, static_cast<float*>(out));
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_upsample2x_add(void* x, const void* up, int n, int h, int w, int c, void* x_relu,
                                              const void* skip, int skip_n, int f16, mivos_stream_t s) {
  const int v = f16 ? 8 : 4;
  MIVOS_REQUIRE(x && up && AL16(x) && AL16(up) && (!x_relu || AL16(x_relu)) && (!skip || AL16(skip)) && c % v == 0 &&
                    h % 2 == 0 && w % 2 == 0,
                "upsample2x_add: bad arguments");
  MIVOS_REQUIRE(!skip || (skip_n >= 1 && n % skip_n == 0), "upsample2x_add: %d skip maps do not divide %d images", skip_n, n);
  const int per_skip = skip ? n / skip_n : 1;
  const int64_t total = static_cast<int64_t>(n) * h * w * (c / v);
  if (f16)
    launch_pdl(upsample2x_add_kernel<__half>, capped_grid(total), kThreads, 0, ST(s), 
        static_cast<__half*>(x), static_cast<const __half*>(up), n, h, w, c / v, static_cast<__half*>(x_relu),
        static_cast<const __half*>(skip), per_skip);
  else
    launch_pdl(upsample2x_add_kernel<float>, capped_grid(total), kThreads, 0, ST(s), 
        static_cast<float*>(x), static_cast<const float*>(up), n, h, w, c / v, static_cast<float*>(x_relu),
        static_cast<const float*>(skip), per_skip);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_halo_copy(const void* src, int src_n, int src_cstride, int src_coff, void* dst,
                                         int dst_cstride, int dst_coff, int n, int h, int w, int c, int relu,
                                         int src_f16, int dst_f16, mivos_stream_t s) {
  MIVOS_REQUIRE(src && dst, "halo_copy: null pointer");
  MIVOS_REQUIRE(c % 4 == 0 && src_coff + c <= src_cstride && dst_coff + c <= dst_cstride && src_n >= 1 && n % src_n == 0,
                "halo_copy: bad channel window");
  const int64_t total = static_cast<int64_t>(n) * h * w * (c / 4);
  const unsigned g = capped_grid(total);
#define HC(TS, TD)                                                                                              \
  launch_pdl(halo_copy_kernel<TS, TD>, g, kThreads, 0, ST(s), static_cast<const TS*>(src), src_n, src_cstride, src_coff, \
                                                      static_cast<TD*>(dst), dst_cstride, dst_coff, n, h, w, c / 4, relu)
  if (src_f16 && dst_f16) HC(__half, __half);
  else if (src_f16) HC(__half, float);
  else if (dst_f16) HC(float, __half);
  else HC(float, float);
#undef HC
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_halo_to_nchw(const void* halo, int n, int h, int w, int cstride, int coff, int c,
                                            float* nchw, int f16, mivos_stream_t s) {
  MIVOS_REQUIRE(halo && nchw && n > 0 && c > 0 && coff + c <= cstride, "halo_to_nchw: bad arguments");
  dim3 grid(ceil_div(h * w, 32), ceil_div(c, 32), n);
  if (f16) launch_pdl(halo_to_nchw_kernel<__half>, grid, 256, 0, ST(s), static_cast<const __half*>(halo), h, w, cstride, coff, c, nchw);
  else launch_pdl(halo_to_nchw_kernel<float>, grid, 256, 0, ST(s), static_cast<const float*>(halo), h, w, cstride, coff, c, nchw);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_nchw_to_halo(const float* nchw, int n, int h, int w, int c, void* halo, int cstride,
                                            int coff, int relu, int f16, mivos_stream_t s) {
  MIVOS_REQUIRE(halo && nchw && n > 0 && c > 0 && coff + c <= cstride, "nchw_to_halo: bad arguments");
  dim3 grid(ceil_div(h * w, 32), ceil_div(c, 32), n);
  if (f16) launch_pdl(nchw_to_halo_kernel<__half>, grid, 256, 0, ST(s), nchw, h, w, c, static_cast<__half*>(halo), cstride, coff, relu);
  else launch_pdl(nchw_to_halo_kernel<float>, grid, 256, 0, ST(s), nchw, h, w, c, static_cast<float*>(halo), cstride, coff, relu);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_fusion_gather(const float* im, const float* seg1, const float* seg2, const float* attn,
                                             float nc, float nr, int h, int w, void* out_halo, int cpad, int f16,
                                             mivos_stream_t s) {
  MIVOS_REQUIRE(im && seg1 && seg2 && attn && out_halo && AL16(out_halo) && cpad >= 9, "fusion_gather: bad arguments");
  const int64_t plane = static_cast<int64_t>(h) * w;
  if (f16)
    launch_pdl(fusion_gather_kernel<__half>, capped_grid(plane), kThreads, 0, ST(s), im, seg1, seg2, attn, nc, nr, h, w, static_cast<__half*>(out_halo), cpad);
  else
    launch_pdl(fusion_gather_kernel<float>, capped_grid(plane), kThreads, 0, ST(s), im, seg1, seg2, attn, nc, nr, h, w, static_cast<float*>(out_halo), cpad);
  MIVOS_LAUNCHED();
  return MIVOS_OK;
}
