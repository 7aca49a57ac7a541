// Implicit-GEMM convolution on the Hopper tensor cores (wgmma, TF32 or FP16 operands, FP32
// accumulate), sm_90a only.
//
// Replaces every nn.Conv2d(+BatchNorm eval)(+ReLU)(+residual) of the reference's propagation
// path: model/propagation/modules.py:15-35 (ResBlock), :38-89 (encoders), :92-114 (Upsample,
// KeyValue), mod_resnet.py:76-112 (Bottleneck), prop_net.py:14-31 (Decoder),
// model/fusion_net.py:8-50 (FusionNet).
//
// Activations live in HALO layout (include/mivos_b200.h): a flattened [rows, C] matrix with a
// zero one-pixel border per image, so tap (dy,dx) of a 3x3/pad-1 conv is the same matrix shifted
// by dy*(W+2)+dx rows.  One CTA computes a 128-row x BN-column output tile (or one K range of it
// under split-K):
//   warpgroup 0 : one thread is the TMA producer - per (tap, 128-byte k-block) it loads the A box
//                 {k-block x 128 rows} at the shifted row and the B box {k-block x BN rows} of the
//                 packed weights, 128B-swizzled, into a ring of STAGES stages
//   warpgroups 1-2 : rows 0-63 / 64-127 of the tile: 4 x wgmma (K = 32 bytes each) per k-block
//                 into a register accumulator; a stage is handed back once the wgmmas that read it
//                 have completed (one arrival per warp)
//   epilogue   : the accumulators are parked in a row-major shared-memory tile (over the drained
//                 ring), then every warp stores 32 x 32 blocks: + bias (+ residual) (ReLU), to
//                 interior rows only (the halo stays zero)
// Roofline: tensor pipe (TF32 / FP16); algorithmic flops = 2 * rows_interior * taps*cin * cout.
#include "host_util.h"
#include "pdl.cuh"
#include "sm90.cuh"

#include <atomic>
#include <stdlib.h>

namespace mivos {
extern std::atomic<int64_t> g_launches;

namespace {

constexpr int BM = 128;
constexpr int BK = 32;  // fp32 elements per k-block = one 128-byte swizzle row
constexpr int A_BYTES = BM * BK * 4;

struct ConvParams {
  int64_t rows;  // HALO rows of the output map
  int n, h, w;
  int in_coff;
  int kblocks;  // cin_pad / bk
  int taps;
  int cout, cout_pad;
  const float* bias;
  float* out;
  int out_cstride, out_coff;
  const float* residual;
  int res_cstride, res_coff;
  float* out_relu;
  int out_relu_cstride, out_relu_coff;
  int relu;
  int round_tf32;
  int f16_in;   // operands are fp16: kind::f16 MMAs, 64 elements per 128-byte k-block
  int f16_out;  // out / residual / out_relu are fp16
  int bk;       // elements per k-block: 32 (fp32) or 64 (fp16)
  int splits;   // split-K: K ranges per output tile (1 = off); partial tiles parked in sk_ws
  float* sk_ws;
  int* sk_cnt;
  int* err;
};

// round-to-nearest (ties away) to TF32 precision: the tensor core reads only the TF32 bits of fp32
// operands (truncation), which would bias every layer by about -1e-3; storing activations
// pre-rounded makes that truncation a no-op.
__device__ __forceinline__ float rna_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

#include "conv_epilogue.cuh"

constexpr int kConvThreads = 384;  // producer warpgroup + two MMA / epilogue warpgroups

template <int BN, int STAGES>
struct SmemLayout {
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  // accumulator tile [128][BN + 8] fp32: the pad makes the fragment stores (8-byte pieces of 4 rows per
  // half-warp) conflict-free; it reuses the ring, which is drained when the tile is written
  static constexpr int ACC_STRIDE = BN + 8;
  static constexpr int ACC_BYTES = BM * ACC_STRIDE * 4;
  static constexpr int BAR_OFF = ((RING_BYTES > ACC_BYTES ? RING_BYTES : ACC_BYTES) + 7) & ~7;
  static constexpr int TOTAL = BAR_OFF + 2 * STAGES * 8;
};

template <int BN, int STAGES, bool F16>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const ConvParams p, const int m_tiles) {
  using L = SmemLayout<BN, STAGES>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // dynamic smem base is only guaranteed 16B aligned; round up to the 1024B the swizzle needs
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + STAGES;

  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int mt = blockIdx.x, nt = blockIdx.y, split = blockIdx.z;
  const int64_t m0 = static_cast<int64_t>(mt) * BM;
  const int n0 = nt * BN;
  const int iters = p.taps * p.kblocks;
  const int S = p.splits;
  const int j0 = static_cast<int>(static_cast<int64_t>(split) * iters / S);
  const int j1 = static_cast<int>(static_cast<int64_t>(split + 1) * iters / S);

  if (threadIdx.x == 0) {
    sm90::prefetch_tmap(&tmA);
    sm90::prefetch_tmap(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      sm90::mbar_init(&full_bar[s], 1);
      sm90::mbar_init(&empty_bar[s], 8);  // one arrival per MMA warp
    }
    sm90::fence_barrier_init();
  }
  __syncthreads();
  // everything above touched only shared memory and the kernel parameters: it ran under the previous
  // kernel's tail (pdl.cuh); from here on global memory is read and written
  pdl_wait();

  if (warp < 4) {
    sm90::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      const int wp = p.w + 2;
      for (int j = j0, it = 0; j < j1; ++j, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        const int t = j / p.kblocks;
        const int kb = j - t * p.kblocks;
        int64_t row = m0;
        if (p.taps == 9) row += static_cast<int64_t>(t / 3 - 1) * wp + (t % 3 - 1);
        else if (p.taps == 4) row += static_cast<int64_t>(t - 2) * wp;  // vertical taps dy = -2..1 (space-to-depth stem)
        sm90::mbar_wait(&empty_bar[s], ph ^ 1, p.err, 101);
        sm90::mbar_arrive_expect_tx(&full_bar[s], L::STAGE_BYTES);
        uint8_t* sa = smem + s * L::STAGE_BYTES;
        sm90::tma_load_2d(sa, &tmA, &full_bar[s], p.in_coff + kb * p.bk, static_cast<int32_t>(row));
        sm90::tma_load_2d(sa + A_BYTES, &tmB, &full_bar[s], kb * p.bk, t * p.cout_pad + n0);
      }
    }
    return;
  }

  sm90::setmaxnreg_inc<232>();
  const int wg = warp / 4 - 1;  // 0: rows 0-63, 1: rows 64-127
  const int tw = threadIdx.x - 128 * (wg + 1);
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  int prev = -1;
  for (int j = j0, it = 0; j < j1; ++j, ++it) {
    const int s = it % STAGES;
    sm90::mbar_wait(&full_bar[s], (it / STAGES) & 1, p.err, 102);
    const uint32_t sa = sm90::smem_u32(smem + s * L::STAGE_BYTES);
    const uint64_t da = sm90::make_desc_sw128(sa + wg * 64 * 128);
    const uint64_t db = sm90::make_desc_sw128(sa + A_BYTES);
    sm90::wgmma_fence();
    // a 128-byte k-block row is 4 MMA K-steps of 32 bytes in either type (8 x fp32 / 16 x fp16): +2 in 16-byte units
#pragma unroll
    for (int k = 0; k < 4; ++k) sm90::wgmma<BN, F16>(acc, da + 2 * k, db + 2 * k, (j != j0 || k != 0) ? 1u : 0u);
    sm90::wgmma_commit();
    sm90::wgmma_wait<1>();  // the previous k-block's wgmmas are done: its stage may be refilled
    if (prev >= 0 && lane == 0) sm90::mbar_arrive(&empty_bar[prev]);
    prev = s;
  }
  sm90::wgmma_wait<0>();
  sm90::fence_acc(acc);

  // both warpgroups have finished reading the ring (and every TMA write into it was waited for): the
  // accumulator tile may overwrite it
  sm90::named_sync(1, 256);
  float* tile = reinterpret_cast<float*>(smem);
  {
    const int r = wg * 64 + (tw >> 5) * 16 + ((tw & 31) >> 2);
    const int c = 2 * (tw & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      *reinterpret_cast<float2*>(tile + r * L::ACC_STRIDE + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(tile + (r + 8) * L::ACC_STRIDE + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  sm90::named_sync(1, 256);

  // epilogue: 32-row x 32-column blocks, consumer warp cw takes blocks cw, cw + 8, ...
  const int cw = warp - 4;
  const int wp = p.w + 2;
  const int64_t per_img = static_cast<int64_t>(p.h + 2) * wp;
#pragma unroll 1
  for (int blk = cw; blk < 4 * (BN / 32); blk += 8) {
    const int rb = blk & 3, cb = blk >> 2;
    const int64_t row0 = m0 + rb * 32;
    const float* src = tile + rb * 32 * L::ACC_STRIDE + cb * 32;
    if (S > 1) {
      // split-K: park the fp32 partial block in the workspace [tile][split][128 rows][BN]; splitk_epilogue_kernel
      // (next launch) sums the S partials in split order and applies bias / residual / ReLU / conversion
      float* dst = p.sk_ws + (((static_cast<int64_t>(nt) * m_tiles + mt) * S + split) * BM + rb * 32) * BN + cb * 32;
      const int c4 = lane & 7, rsub = lane >> 3;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = i * 4 + rsub;
        *reinterpret_cast<float4*>(dst + rr * BN + c4 * 4) = *reinterpret_cast<const float4*>(src + rr * L::ACC_STRIDE + c4 * 4);
      }
      continue;
    }
    const int64_t r = row0 + lane;
    bool interior = false;
    if (r < p.rows) {
      const int64_t rem = r % per_img;
      const int y = static_cast<int>(rem / wp);
      const int x = static_cast<int>(rem - static_cast<int64_t>(y) * wp);
      interior = (y >= 1) && (y <= p.h) && (x >= 1) && (x <= p.w);
    }
    const uint32_t interior_mask = __ballot_sync(0xffffffffu, interior);
    conv_epilogue_block(src, L::ACC_STRIDE, lane, row0, interior_mask, n0 + cb * 32, p);
  }
}

// Split-K second pass: out = epilogue(sum over the S parked partial tiles, in split order).
// Partials are [tile = nt * m_tiles + mt][split][128 rows][bn] fp32 (tile order of tile_of<1>);
// a thread owns one output row and 4 consecutive channels: reads are 16-byte pieces of 128-byte
// row segments, consecutive threads consecutive channels.
__global__ void splitk_epilogue_kernel(const ConvParams p, const int bn) {
  pdl_prologue();
  const int S = p.splits;
  const int cq = p.cout_pad / 4;
  const int m_tiles = static_cast<int>((p.rows + BM - 1) / BM);
  const int wp = p.w + 2;
  const int64_t per_img = static_cast<int64_t>(p.h + 2) * wp;
  const int64_t work = p.rows * cq;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < work;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t row = i / cq;
    const int col = static_cast<int>(i - row * cq) * 4;
    if (col >= p.cout) continue;
    const int64_t rem = row % per_img;
    const int y = static_cast<int>(rem / wp), x = static_cast<int>(rem - static_cast<int64_t>(y) * wp);
    if (y < 1 || y > p.h || x < 1 || x > p.w) continue;  // halo rows are never written
    const int mt = static_cast<int>(row / BM), nt = col / bn;
    const int64_t tile = static_cast<int64_t>(nt) * m_tiles + mt;
    const float* src = p.sk_ws + ((tile * S) * BM + (row - static_cast<int64_t>(mt) * BM)) * bn + (col - nt * bn);
    float4 acc = *reinterpret_cast<const float4*>(src);
    for (int sp = 1; sp < S; ++sp) {
      const float4 t = *reinterpret_cast<const float4*>(src + static_cast<int64_t>(sp) * BM * bn);
      acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
    }
    float o[4] = {acc.x, acc.y, acc.z, acc.w};
    const int nvalid = p.cout - col < 4 ? p.cout - col : 4;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (e >= nvalid) break;
      const int c = col + e;
      float v = o[e] + p.bias[c];
      if (p.f16_out) {
        if (p.residual) v += __half2float(reinterpret_cast<const __half*>(p.residual)[row * p.res_cstride + p.res_coff + c]);
        if (p.relu) v = fmaxf(v, 0.f);
        reinterpret_cast<__half*>(p.out)[row * p.out_cstride + p.out_coff + c] = __float2half_rn(v);
        if (p.out_relu)
          reinterpret_cast<__half*>(p.out_relu)[row * p.out_relu_cstride + p.out_relu_coff + c] = __float2half_rn(fmaxf(v, 0.f));
      } else {
        if (p.residual) v += p.residual[row * p.res_cstride + p.res_coff + c];
        if (p.relu) v = fmaxf(v, 0.f);
        if (p.round_tf32) v = rna_tf32(v);
        p.out[row * p.out_cstride + p.out_coff + c] = v;
        if (p.out_relu) p.out_relu[row * p.out_relu_cstride + p.out_relu_coff + c] = fmaxf(v, 0.f);
      }
    }
  }
}

template <int BN, int STAGES, bool F16>
int launch(const mivos_conv_args* a, const ConvParams& p, cudaStream_t stream) {
  using L = SmemLayout<BN, STAGES>;
  constexpr int smem_bytes = L::TOTAL + 1024;  // slack for the manual 1024B alignment
  static_assert(smem_bytes <= 232448, "stage ring exceeds the 227 KB a CTA may use");
  auto kernel = conv_gemm_kernel<BN, STAGES, F16>;
  static bool configured = false;
  if (!configured) {
    MIVOS_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    configured = true;
  }
  CUtensorMap tmA, tmB;
  const int eb = a->in_f16 ? 2 : 4;
  int rc = encode_tmap_2d(&tmA, a->in, static_cast<uint64_t>(a->in_rows), static_cast<uint64_t>(a->in_cstride),
                          static_cast<uint64_t>(a->in_cstride), p.bk, BM, eb);
  if (rc != MIVOS_OK) return rc;
  rc = encode_tmap_2d(&tmB, a->weight, static_cast<uint64_t>(a->taps) * a->cout_pad, static_cast<uint64_t>(a->cin_pad),
                      static_cast<uint64_t>(a->cin_pad), p.bk, BN, eb);
  if (rc != MIVOS_OK) return rc;
  const int m_tiles = static_cast<int>(ceil_div64(p.rows, BM));
  dim3 grid(static_cast<unsigned>(m_tiles), static_cast<unsigned>(a->cout_pad / BN), static_cast<unsigned>(p.splits));
  MIVOS_CUDA_OK(launch_pdl(kernel, grid, kConvThreads, smem_bytes, stream, tmA, tmB, p, m_tiles));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return MIVOS_OK;
}

}  // namespace
}  // namespace mivos

using namespace mivos;

namespace mivos {
std::atomic<int> g_tile_override{0};
}

namespace mivos {
namespace {
// Tile width BN in {256,128,64,32} (must divide cout_pad) and split-K factor by a small cost model
// (tools/tile_sweep.py measures the tile widths on the device), in KB-equivalents of shared-memory
// ingest, the resource that bounds the main loop:
//   main loop of a tile = k-blocks x (16 KB of A + BN/8 KB of B + 6 KB fixed barrier/issue cost)
//   epilogue of a tile  = half its output KB (+ the same again per residual read / ReLU copy)
//   the tiles run in ceil(tiles / SMs) waves of one CTA per SM; the cost of a wave is the larger of the two
//   terms (the CTAs of a wave are at different phases), plus the smaller one once for the last wave.
// Pure host arithmetic on the argument block (no pointer is dereferenced, no device is touched):
// exported as mivos_conv_plan so the choice can be unit-tested without a GPU.
constexpr int64_t kSkCounterBytes = 65536;  // reserved head of the split-K workspace

int plan_tiles(const mivos_conv_args* a, const int sms, int* bn_out, int* splits_out) {
  const int bk = a->in_f16 ? 64 : 32;
  const int64_t rows = static_cast<int64_t>(a->n) * (a->h + 2) * (a->w + 2);
  const int kblocks = a->cin_pad / bk;
  const int64_t mtiles = ceil_div64(rows, BM);
  const double kb_total = static_cast<double>(a->taps) * kblocks;
  const double out_kb_per_col = (a->out_f16 ? 0.125 : 0.25) * (1.0 + (a->residual ? 1.0 : 0.0) + (a->out_relu ? 1.0 : 0.0));
  // Split-K (S > 1): when the row tiles of a small map cannot fill the SMs, S CTAs share a tile's K
  // range, so a wide tile (few operand re-reads) still runs on all SMs.  Costs: the fp32 partials
  // through L2 and a second (HBM-bound, PDL-chained) launch that sums them and applies the
  // epilogue, ~8 us = 700 KB-equivalents — it pays only for the K >= 9 x 512 layers of the
  // 1/16-resolution maps.  Needs the caller's workspace.
  static const bool allow_splitk = [] {  // MIVOS_CONV_SPLITK=0: A/B measurements
    const char* e = getenv("MIVOS_CONV_SPLITK");
    return !(e && e[0] == '0');
  }();
  int bn = 32, splits = 1;
  double best_cost = 1e300;
  const int iters_total = a->taps * kblocks;
  for (int cand = 256; cand >= 32; cand >>= 1) {
    if (a->cout_pad % cand) continue;
    const int64_t tiles = mtiles * (a->cout_pad / cand);
    for (int sp = 1; sp <= 8; ++sp) {
      if (sp > 1) {
        if (!allow_splitk || !a->splitk_ws || iters_total / sp < 4 || tiles * sp > 2 * sms || tiles > kSkCounterBytes / 4) break;
        if (kSkCounterBytes + tiles * sp * BM * cand * 4 > a->splitk_ws_bytes) break;
      }
      const double rounds = static_cast<double>((tiles * sp + sms - 1) / sms);
      const double ml = kb_total / sp * (16.0 + cand / 8.0 + 6.0);
      // epilogue of a tile: half a KB-equivalent per output KB (fitted to an H100 sweep of the fp16 cfg-2 layers,
      // tools/tile_sweep.py: every layer within 5 % of its best tile width)
      const double ep = cand * out_kb_per_col;
      double cost = rounds * (ml > ep ? ml : ep) + (ml > ep ? ep : ml);
      if (sp > 1) cost = (ml + cand * 0.5 + 700.0) * 1.15;  // + partial write + reduce launch; must win by a margin
      if (cost < best_cost) {  // ties keep the wider tile (fewer barrier round trips per flop)
        best_cost = cost;
        bn = cand;
        splits = sp;
      }
    }
  }
  const int forced = g_tile_override.load(std::memory_order_relaxed);
  if (forced > 0) {
    MIVOS_REQUIRE((forced == 32 || forced == 64 || forced == 128 || forced == 256) && a->cout_pad % forced == 0,
                  "conv_gemm: tile override %d does not divide cout_pad %d", forced, a->cout_pad);
    bn = forced;
    splits = 1;
  }
  *bn_out = bn;
  *splits_out = splits;
  return MIVOS_OK;
}

}  // namespace
}  // namespace mivos

extern "C" MIVOS_API int mivos_conv_plan(const mivos_conv_args* a, int sms, int* bn, int* splits) {
  MIVOS_REQUIRE(a && bn && splits, "conv_plan: null pointer");
  MIVOS_REQUIRE((a->taps == 1 || a->taps == 4 || a->taps == 9) && a->cin_pad > 0 && a->cin_pad % (a->in_f16 ? 64 : 32) == 0 &&
                    a->cout_pad > 0 && a->cout_pad % 32 == 0 && a->n > 0 && a->h > 0 && a->w > 0,
                "conv_plan: bad shape");
  return plan_tiles(a, sms > 0 ? sms : num_sms(), bn, splits);
}

extern "C" MIVOS_API int mivos_conv_tile_override(int bn) {
  mivos::g_tile_override.store(bn, std::memory_order_relaxed);
  return MIVOS_OK;
}

extern "C" MIVOS_API int mivos_conv_gemm(const mivos_conv_args* a, mivos_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MIVOS_REQUIRE(a && a->in && a->weight && a->bias && a->out, "conv_gemm: null pointer");
  MIVOS_REQUIRE(a->taps == 1 || a->taps == 4 || a->taps == 9, "conv_gemm: taps must be 1, 4 or 9 (got %d)", a->taps);
  const int bk = a->in_f16 ? 64 : 32;
  const int ea = a->in_f16 ? 8 : 4, eo = a->out_f16 ? 8 : 4;  // elements per 16 bytes
  MIVOS_REQUIRE(a->cin_pad > 0 && a->cin_pad % bk == 0, "conv_gemm: cin_pad %% %d != 0 (%d)", bk, a->cin_pad);
  MIVOS_REQUIRE(a->cout_pad > 0 && a->cout_pad % 32 == 0 && a->cout <= a->cout_pad && a->cout > 0,
                "conv_gemm: bad cout/cout_pad (%d/%d)", a->cout, a->cout_pad);
  MIVOS_REQUIRE(a->in_cstride % ea == 0 && a->in_coff % ea == 0 && a->in_coff + a->cin_pad <= a->in_cstride,
                "conv_gemm: input channel window [%d,+%d) does not fit stride %d", a->in_coff, a->cin_pad, a->in_cstride);
  MIVOS_REQUIRE(a->out_cstride % eo == 0 && a->out_coff % eo == 0, "conv_gemm: out stride/offset must be multiples of %d", eo);
  MIVOS_REQUIRE(!a->residual || (a->res_cstride % eo == 0 && a->res_coff % eo == 0), "conv_gemm: residual stride/offset must be multiples of %d", eo);
  MIVOS_REQUIRE(!a->out_relu || (a->out_relu_cstride % eo == 0 && a->out_relu_coff % eo == 0), "conv_gemm: out_relu stride/offset must be multiples of %d", eo);
  MIVOS_REQUIRE((reinterpret_cast<uintptr_t>(a->in) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->weight) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(a->out) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->bias) & 15) == 0,
                "conv_gemm: pointers must be 16-byte aligned");
  MIVOS_REQUIRE(a->n > 0 && a->h > 0 && a->w > 0, "conv_gemm: bad map dims");

  ConvParams p;
  p.rows = static_cast<int64_t>(a->n) * (a->h + 2) * (a->w + 2);
  p.n = a->n; p.h = a->h; p.w = a->w;
  p.in_coff = a->in_coff;
  p.kblocks = a->cin_pad / bk;
  p.bk = bk;
  p.f16_in = a->in_f16 ? 1 : 0;
  p.f16_out = a->out_f16 ? 1 : 0;
  p.taps = a->taps;
  p.cout = a->cout; p.cout_pad = a->cout_pad;
  p.bias = a->bias;
  p.out = static_cast<float*>(a->out); p.out_cstride = a->out_cstride; p.out_coff = a->out_coff;
  p.residual = static_cast<const float*>(a->residual); p.res_cstride = a->res_cstride; p.res_coff = a->res_coff;
  p.out_relu = static_cast<float*>(a->out_relu); p.out_relu_cstride = a->out_relu_cstride; p.out_relu_coff = a->out_relu_coff;
  p.relu = a->relu & 1;
  p.round_tf32 = (a->relu >> 1) & 1;
  p.err = device_error_flag();
  MIVOS_REQUIRE(p.rows < (1ll << 31) - 4096, "conv_gemm: too many rows for int32 TMA coordinates");

  int bn = 32, splits = 1;
  {
    const int rc = plan_tiles(a, num_sms(), &bn, &splits);
    if (rc != MIVOS_OK) return rc;
  }
  p.splits = splits;
  p.sk_cnt = nullptr;
  p.sk_ws = reinterpret_cast<float*>(static_cast<uint8_t*>(a->splitk_ws) + kSkCounterBytes);

  int rc = MIVOS_OK;
  switch (bn) {
    // stage counts: a ring of ~190 KB of 128-byte k-block stages (one CTA per SM)
    case 256: rc = a->in_f16 ? launch<256, 4, true>(a, p, stream) : launch<256, 4, false>(a, p, stream); break;
    case 128: rc = a->in_f16 ? launch<128, 6, true>(a, p, stream) : launch<128, 6, false>(a, p, stream); break;
    case 64:  rc = a->in_f16 ? launch<64, 8, true>(a, p, stream) : launch<64, 8, false>(a, p, stream); break;
    default:  rc = a->in_f16 ? launch<32, 9, true>(a, p, stream) : launch<32, 9, false>(a, p, stream); break;
  }
  if (rc != MIVOS_OK || p.splits == 1) return rc;
  // split-K second pass: one thread per (row, 4 channels)
  const int64_t work = p.rows * (a->cout_pad / 4);
  int64_t grid = (work + 255) / 256;
  if (grid > num_sms() * 32ll) grid = num_sms() * 32ll;
  MIVOS_CUDA_OK(launch_pdl(splitk_epilogue_kernel, static_cast<unsigned>(grid), 256, 0, stream, p, bn));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return MIVOS_OK;
}
