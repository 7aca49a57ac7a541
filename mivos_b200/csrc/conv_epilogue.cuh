// Epilogue of the implicit-GEMM convolution kernel: one 128-row x BN-column output tile, straight from the
// wgmma accumulator fragments of the two MMA warpgroups.
//
// Each thread applies  o = acc + bias, (+ residual), (ReLU), then the rounding (fp16 RNE / TF32 RNA)  to its own
// fragment elements and writes the result in fragment order into a row-padded staging tile.  With a residual the
// staging tile IS the residual tile the producer warpgroup prefetched with bulk copies: every element is read and
// overwritten by the same thread.  Then every interior row segment goes to global memory as one bulk copy.  Border
// rows are never read or written.  A row segment's bytes past its last multiple of 16 (a channel count such as 1,
// 36 or 100 fp16 channels) cannot be a bulk copy: those channels go element-wise through the staging tile.
#pragma once
#include <cuda_fp16.h>

// Row r of the output map is an interior pixel (not in the zero HALO border, not past the last row).
__device__ __forceinline__ bool conv_row_interior(const ConvParams& p, const int64_t r) {
  if (r >= p.rows) return false;
  const int wp = p.w + 2;
  const int64_t rem = r % (static_cast<int64_t>(p.h + 2) * wp);
  const int y = static_cast<int>(rem / wp);
  const int x = static_cast<int>(rem - static_cast<int64_t>(y) * wp);
  return y >= 1 && y <= p.h && x >= 1 && x <= p.w;
}

// Real output channels of the tile at n0, and how many of them the bulk copies move (the largest count whose
// bytes are a multiple of 16).
__device__ __forceinline__ int conv_tile_cols(const ConvParams& p, const int bn, const int n0) {
  const int c = p.cout - n0;
  return c < 0 ? 0 : (c < bn ? c : bn);
}
__device__ __forceinline__ int conv_bulk_cols(const ConvParams& p, const int ncols) {
  const int esz = p.f16_out ? 2 : 4;
  return ((ncols * esz) & ~15) / esz;
}

// Staging tile row stride in elements: 16 bytes of pad put the 8 rows of a fragment access in different banks.
template <int BN>
constexpr int kStageStride = BN + 8;

// Producer side (one warp): bulk-load the residual segments of the tile's interior rows into the staging tile,
// completing on res_bar.
template <int BN>
__device__ __forceinline__ void conv_prefetch_residual(uint8_t* stile, uint64_t* res_bar, const int lane, const int64_t m0,
                                                       const int n0, const ConvParams& p) {
  const int esz = p.f16_out ? 2 : 4;
  const uint32_t bytes = conv_bulk_cols(p, conv_tile_cols(p, BN, n0)) * esz;
  bool in[4];
  int cnt = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    in[i] = bytes > 0 && conv_row_interior(p, m0 + lane + 32 * i);
    cnt += in[i] ? 1 : 0;
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if (lane == 0) sm90::mbar_arrive_expect_tx(res_bar, cnt * bytes);
  __syncwarp();
  const uint8_t* src = reinterpret_cast<const uint8_t*>(p.residual);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (!in[i]) continue;
    const int r = lane + 32 * i;
    sm90::bulk_load(stile + static_cast<int64_t>(r) * kStageStride<BN> * esz,
                    src + ((m0 + r) * p.res_cstride + p.res_coff + n0) * esz, bytes, res_bar);
  }
}

// Fragment pass: o = acc + bias (+ residual from the staging tile) (ReLU) (rounding) into the staging tile, every
// column of the tile.  Templated on the output type and the residual, with ReLU / rounding as selects, so the fully
// unrolled body stays small: it is straight-line code run once per tile, and a large one is paid in instruction
// fetches.
template <int BN, bool F16OUT, bool RES>
__device__ __forceinline__ void conv_epilogue_frags(const float (&acc)[BN / 2], uint8_t* stile, const int r0, const int cq,
                                                    const int n0, const ConvParams& p) {
  constexpr int STRIDE = kStageStride<BN>;
  const bool relu = p.relu != 0, rnd = !F16OUT && p.round_tf32;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int c = 8 * j + cq;
    const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + c));
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int e = (r0 + 8 * hf) * STRIDE + c;
      float o0 = acc[4 * j + 2 * hf] + b.x, o1 = acc[4 * j + 2 * hf + 1] + b.y;
      if constexpr (RES) {
        const float2 rv = F16OUT ? __half22float2(*reinterpret_cast<const __half2*>(reinterpret_cast<__half*>(stile) + e))
                                 : *reinterpret_cast<const float2*>(reinterpret_cast<float*>(stile) + e);
        o0 += rv.x;
        o1 += rv.y;
      }
      o0 = relu ? fmaxf(o0, 0.f) : o0;
      o1 = relu ? fmaxf(o1, 0.f) : o1;
      if constexpr (F16OUT) {
        *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(stile) + e) = __floats2half2_rn(o0, o1);
      } else {
        const float t0 = rna_tf32(o0), t1 = rna_tf32(o1);
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(stile) + e) = make_float2(rnd ? t0 : o0, rnd ? t1 : o1);
      }
    }
  }
}

// max(v, 0) of a stored output value: the conversion of max(o, 0), since rounding is monotonic and keeps 0 (a
// half is > 0 exactly where o > 0 rounds to a non-zero value)
__device__ __forceinline__ float conv_relu_of_stored(const float v) { return v > 0.f ? v : 0.f; }

// Consumer side: called by all 256 threads of the MMA warpgroups (tw = thread within warpgroup wg) once the ring is
// drained.  Accumulator fragment: rows wg*64 + 16*(tw/32) + (tw%32)/4 (+8), columns 8j + 2*(tw%4) (+1).
template <int BN>
__device__ __forceinline__ void conv_epilogue_tile(const float (&acc)[BN / 2], uint8_t* stile, uint64_t* res_bar,
                                                   const int wg, const int tw, const int64_t m0, const int n0,
                                                   const ConvParams& p) {
  constexpr int STRIDE = kStageStride<BN>;
  const int esz = p.f16_out ? 2 : 4;
  const int ncols = conv_tile_cols(p, BN, n0);
  const int nbulk = conv_bulk_cols(p, ncols);
  const int ntail = ncols - nbulk;  // channels past the bulk copies: element-wise, through the staging tile
  const int t = wg * 128 + tw;
  __half* const sh = reinterpret_cast<__half*>(stile);
  float* const sf = reinterpret_cast<float*>(stile);
  if (p.residual) {
    sm90::mbar_wait(res_bar, 0, p.err, 104);
    if (ntail > 0) {
      for (int k = t; k < BM * ntail; k += 256) {
        const int r = k / ntail, c = nbulk + k % ntail;
        if (!conv_row_interior(p, m0 + r)) continue;
        const int64_t off = (m0 + r) * p.res_cstride + p.res_coff + n0 + c;
        if (p.f16_out) sh[r * STRIDE + c] = reinterpret_cast<const __half*>(p.residual)[off];
        else sf[r * STRIDE + c] = p.residual[off];
      }
      sm90::named_sync(1, 256);
    }
  }
  const int r0 = wg * 64 + (tw >> 5) * 16 + ((tw & 31) >> 2);
  const int cq = 2 * (tw & 3);
  if (p.f16_out) {
    if (p.residual) conv_epilogue_frags<BN, true, true>(acc, stile, r0, cq, n0, p);
    else conv_epilogue_frags<BN, true, false>(acc, stile, r0, cq, n0, p);
  } else {
    if (p.residual) conv_epilogue_frags<BN, false, true>(acc, stile, r0, cq, n0, p);
    else conv_epilogue_frags<BN, false, false>(acc, stile, r0, cq, n0, p);
  }

  // threads 0-127 each store one row segment
  const bool store_row = t < BM && nbulk > 0 && conv_row_interior(p, m0 + t);
  const uint32_t bytes = nbulk * esz;
  const uint8_t* srow = stile + static_cast<int64_t>(t) * STRIDE * esz;
  sm90::fence_proxy_async_smem();
  sm90::named_sync(1, 256);
  if (store_row) {
    sm90::bulk_store(reinterpret_cast<uint8_t*>(p.out) + ((m0 + t) * p.out_cstride + p.out_coff + n0) * esz, srow, bytes);
    sm90::bulk_commit();
  }
  for (int k = t; k < BM * ntail; k += 256) {
    const int r = k / ntail, c = nbulk + k % ntail;
    if (!conv_row_interior(p, m0 + r)) continue;
    const int64_t oo = (m0 + r) * p.out_cstride + p.out_coff + n0 + c;
    const int64_t ro = (m0 + r) * p.out_relu_cstride + p.out_relu_coff + n0 + c;
    if (p.f16_out) {
      const __half v = sh[r * STRIDE + c];
      reinterpret_cast<__half*>(p.out)[oo] = v;
      if (p.out_relu) reinterpret_cast<__half*>(p.out_relu)[ro] = __float2half_rn(conv_relu_of_stored(__half2float(v)));
    } else {
      const float v = sf[r * STRIDE + c];
      p.out[oo] = v;
      if (p.out_relu) p.out_relu[ro] = fmaxf(v, 0.f);
    }
  }
  if (p.out_relu && nbulk > 0) {
    // the ReLU copy is made in place once the primary store (and the tail above) has read the staging tile
    if (store_row) sm90::bulk_wait_read0();
    sm90::named_sync(1, 256);
    const int nch = nbulk * esz / 16;
    for (int k = t; k < BM * nch; k += 256) {
      uint4* q = reinterpret_cast<uint4*>(stile + (k / nch) * STRIDE * esz + (k % nch) * 16);
      uint4 v = *q;
      uint32_t* w = reinterpret_cast<uint32_t*>(&v);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (p.f16_out) {
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
          const __half2 h = __floats2half2_rn(conv_relu_of_stored(f.x), conv_relu_of_stored(f.y));
          w[i] = *reinterpret_cast<const uint32_t*>(&h);
        } else {
          w[i] = __float_as_uint(fmaxf(__uint_as_float(w[i]), 0.f));
        }
      }
      *q = v;
    }
    sm90::fence_proxy_async_smem();
    sm90::named_sync(1, 256);
    if (store_row) {
      sm90::bulk_store(reinterpret_cast<uint8_t*>(p.out_relu) + ((m0 + t) * p.out_relu_cstride + p.out_relu_coff + n0) * esz,
                       srow, bytes);
      sm90::bulk_commit();
    }
  }
  // the shared memory a bulk store reads must outlive the read
  if (store_row) sm90::bulk_wait_read0();
}
