// Epilogue of the implicit-GEMM convolution kernel: one 32-row x 32-column block of the fp32
// accumulator tile per warp per call.
//
// The MMA warpgroups park their accumulator fragments in a row-major shared-memory tile; the
// epilogue reads it back segment-wise, so all global traffic — residual read, primary store,
// optional ReLU copy — is issued as full row segments: a warp instruction covers 4 rows x 32
// contiguous channels.  The residual segments of the whole block (8 independent loads per lane)
// are requested BEFORE the accumulator reads, so their L2/HBM latency overlaps them instead of
// being paid once per row group.
#pragma once
#include <cuda_fp16.h>

// acc      : the accumulator tile in shared memory, row r of this block at acc[r * stride]
// interior : ballot mask over the warp's 32 rows (bit r set = row row0+r is an interior pixel)
// ncol0    : absolute output channel of column 0 of this block
__device__ __forceinline__ void conv_epilogue_block(const float* acc, const int stride, const int lane,
                                                    const int64_t row0, const uint32_t interior,
                                                    const int ncol0, const ConvParams& p) {
  const int nvalid = p.cout - ncol0;  // real output channels in this block (warp-uniform)
  if (nvalid <= 0 || interior == 0u) return;
  const int c4 = lane & 7;            // which 4-channel piece of the 32-channel row segment
  const int rsub = lane >> 3;         // 0..3: row within the group of 4 rows one instruction covers
  const bool full = nvalid >= 32;

  if (full) {
    float4 res[8];
    if (p.residual) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = i * 4 + rsub;
        res[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if ((interior >> rr) & 1u) {
          const int64_t off = (row0 + rr) * p.res_cstride + p.res_coff + ncol0 + c4 * 4;
          if (p.f16_out) {
            const uint2 u = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(p.residual) + off));
            const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
            const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
            res[i] = make_float4(lo.x, lo.y, hi.x, hi.y);
          } else {
            res[i] = __ldg(reinterpret_cast<const float4*>(p.residual + off));
          }
        }
      }
    }
    const float4 b = *reinterpret_cast<const float4*>(p.bias + ncol0 + c4 * 4);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int rr = i * 4 + rsub;
      if (!((interior >> rr) & 1u)) continue;
      const float4 a = *reinterpret_cast<const float4*>(acc + rr * stride + c4 * 4);
      const int64_t row = row0 + rr;
      float4 o = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
      if (p.residual) {
        o.x += res[i].x; o.y += res[i].y; o.z += res[i].z; o.w += res[i].w;
      }
      if (p.relu) {
        o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f);
      }
      if (p.f16_out) {
        // fp16 HALO output: round-to-nearest-even conversion, 8-byte stores (64 B per row segment)
        __half2 h01 = __floats2half2_rn(o.x, o.y), h23 = __floats2half2_rn(o.z, o.w);
        uint2 u;
        u.x = *reinterpret_cast<uint32_t*>(&h01);
        u.y = *reinterpret_cast<uint32_t*>(&h23);
        *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(p.out) + row * p.out_cstride + p.out_coff + ncol0 + c4 * 4) = u;
        if (p.out_relu) {
          h01 = __floats2half2_rn(fmaxf(o.x, 0.f), fmaxf(o.y, 0.f));
          h23 = __floats2half2_rn(fmaxf(o.z, 0.f), fmaxf(o.w, 0.f));
          u.x = *reinterpret_cast<uint32_t*>(&h01);
          u.y = *reinterpret_cast<uint32_t*>(&h23);
          *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(p.out_relu) + row * p.out_relu_cstride + p.out_relu_coff + ncol0 + c4 * 4) = u;
        }
        continue;
      }
      if (p.round_tf32) {
        o.x = rna_tf32(o.x); o.y = rna_tf32(o.y); o.z = rna_tf32(o.z); o.w = rna_tf32(o.w);
      }
      *reinterpret_cast<float4*>(p.out + row * p.out_cstride + p.out_coff + ncol0 + c4 * 4) = o;
      if (p.out_relu) {
        const float4 o2 = make_float4(fmaxf(o.x, 0.f), fmaxf(o.y, 0.f), fmaxf(o.z, 0.f), fmaxf(o.w, 0.f));
        *reinterpret_cast<float4*>(p.out_relu + row * p.out_relu_cstride + p.out_relu_coff + ncol0 + c4 * 4) = o2;
      }
    }
    return;
  }
  // ragged channel tail (e.g. decoder.pred: one real output channel): element-wise
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rr = i * 4 + rsub;
    if (!((interior >> rr) & 1u)) continue;
    const int64_t row = row0 + rr;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = c4 * 4 + e;
      if (c < nvalid) {
        float o = acc[rr * stride + c] + p.bias[ncol0 + c];
        if (p.f16_out) {
          if (p.residual) o += __half2float(reinterpret_cast<const __half*>(p.residual)[row * p.res_cstride + p.res_coff + ncol0 + c]);
          if (p.relu) o = fmaxf(o, 0.f);
          reinterpret_cast<__half*>(p.out)[row * p.out_cstride + p.out_coff + ncol0 + c] = __float2half_rn(o);
          if (p.out_relu)
            reinterpret_cast<__half*>(p.out_relu)[row * p.out_relu_cstride + p.out_relu_coff + ncol0 + c] = __float2half_rn(fmaxf(o, 0.f));
          continue;
        }
        if (p.residual) o += p.residual[row * p.res_cstride + p.res_coff + ncol0 + c];
        if (p.relu) o = fmaxf(o, 0.f);
        if (p.round_tf32) o = rna_tf32(o);
        p.out[row * p.out_cstride + p.out_coff + ncol0 + c] = o;
        if (p.out_relu) p.out_relu[row * p.out_relu_cstride + p.out_relu_coff + ncol0 + c] = fmaxf(o, 0.f);
      }
    }
  }
}
