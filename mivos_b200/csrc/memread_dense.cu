// Dense memory read: EvalMemoryReader.forward with top_k=None (reference prop_net.py:99-102), the original STM
// read — softmax over ALL live bank slots, then the value read-out:
//     out[o, q, :] = sum_s softmax_s( key[o,s,:] . (qk[set(o),q,:] / sqrt(128)) ) * value[o,s,:]
// without materialising the [slots, hw] affinity (flash-attention style online softmax over the memory axis).
//
// Pass 1 `memread_dense_kernel`: one CTA per (query tile of 64, chunk of the memory axis, object), 8 warps.
//   The CTA walks its chunk in tiles of 32 slots; key and value rows of the next tile stream into shared memory
//   (cp.async, double-buffered, rows past the live count zero-filled — never loaded) while the current one is used:
//     S  = Q.K^T     on the tensor cores (mma.sync m16n8k8 TF32) in 3xTF32: q_hi.k_hi + q_hi.k_lo + q_lo.k_hi,
//                    fp32 accumulation — hi = cvt.rna(x), lo = cvt.rna(x - hi), formed from the fp32 operands
//                    in shared memory, so the scores carry fp32-level error (a softmax turns a score error d into
//                    a relative weight error of ~d; single-pass TF32 would be ~2^-10 * sum|q.k|)
//     online softmax (4 threads per query row): running max m, running sum l, rescale factor
//                    alpha = exp(m_old - m_new) applied to the O accumulator before the tile's product;
//                    P = exp(s - m) rounded to TF32 (cvt.rna), columns past the live count are -inf (P = 0)
//     O += P.V       mma.sync TF32, warp w owns value channels [64w, 64w + 64) of all 64 queries (128 fp32
//                    accumulators per thread).  The B fragment of m16n8k8 is two scalars per thread, so it is
//                    read straight from the SLOT-major value tile (row stride 520 floats: conflict-free) — no
//                    K-major rewrite of the value tile is needed (wgmma's TF32 form only takes K-major operands).
//   It writes its partial (m, l, O[512]) per query.
// Pass 2 `memread_dense_combine_kernel` (PDL-chained): one warp per (object, query) merges the live chunks in
//   ascending order — M = max m_c, L = sum e^(m_c - M) l_c, O = sum e^(m_c - M) O_c — and writes O / L into the
//   output window (HALO channel block or pixel-major, fp32 or fp16), like the top-k read.
//
// Partition invariant: the chunk length depends on hw ONLY (dense_chunk_tiles), never on the live slot count,
// the device-side count, the bank capacity, the object count or q_div.  So an eager read with slots = n, a
// graph-sized read with *dyn_slots = n, one q_div call for C clips and the C per-clip calls, and two runs of
// one call, give the same bits; the capacity only sizes the grid (chunks past the live count exit at once).
#include "host_util.h"
#include "pdl.cuh"
#include "memread.h"

#include <atomic>

namespace mivos {
extern std::atomic<int64_t> g_launches;
namespace {

constexpr int DQ = 64;          // queries per CTA
constexpr int DS = 32;          // bank slots per tile
constexpr int D_THREADS = 256;  // 8 warps
constexpr int QSTR = 132;       // query / key row stride (floats): conflict-free fragment loads
constexpr int VSTR = 520;       // value row stride: 520 = 8 mod 32, conflict-free B-fragment loads by slot
constexpr int PSTR = 36;        // score / P row stride

struct DenseSmem {
  float q[DQ][QSTR];        // q / sqrt(128), fp32 (split into hi / lo at fragment load)
  float k[2][DS][QSTR];     // key tiles
  float v[2][DS][VSTR];     // value tiles, slot-major as in the bank
  float p[DQ][PSTR];        // scores, then P (TF32-rounded)
  float alpha[DQ];          // rescale factor of the tile, per query
};

struct DenseParams {
  MemreadArgs a;
  int chunk_tiles, chunks;
  float* part_o;   // [K][chunks][hw][512]
  float2* part_ml; // [K][chunks][hw] {m, l}
};

__device__ __forceinline__ uint32_t tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
  return r;
}
// x = hi + lo exactly (hi has 11 significant bits, x - hi is exact in fp32); lo is passed on rounded to TF32
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = tf32_rna(x);
  lo = tf32_rna(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))),
               "l"(gmem), "r"(valid ? 16 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

__global__ void __launch_bounds__(D_THREADS, 1) memread_dense_kernel(const DenseParams p) {
  mivos::pdl_prologue();
  extern __shared__ __align__(16) uint8_t dense_smem[];
  DenseSmem& sm = *reinterpret_cast<DenseSmem*>(dense_smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;  // mma fragment coordinates
  const int q0 = blockIdx.x * DQ;
  const int chunk = blockIdx.y;
  const int obj = blockIdx.z;
  const int64_t n_live = live_slots(p.a, obj);
  const int64_t live_tiles = (n_live + DS - 1) / DS;
  const int64_t t_begin = static_cast<int64_t>(chunk) * p.chunk_tiles;
  if (t_begin >= live_tiles) return;  // chunk past the live bank: the combine does not read it
  int64_t t_end = t_begin + p.chunk_tiles;
  if (t_end > live_tiles) t_end = live_tiles;
  const int ntiles = static_cast<int>(t_end - t_begin);

  const float* keys = p.a.bank_k + static_cast<int64_t>(obj) * p.a.slots_cap * 128;
  const float* vals = p.a.bank_v + static_cast<int64_t>(obj) * p.a.slots_cap * 512;
  auto load_tile = [&](int stage, int64_t tile) {
    const int64_t s0 = tile * DS;
    for (int i = tid; i < DS * 32; i += D_THREADS) {  // 32 rows x 32 float4 of keys
      const int r = i >> 5, c4 = i & 31;
      const bool ok = s0 + r < n_live;
      cp_async16(&sm.k[stage][r][c4 * 4], keys + (ok ? (s0 + r) * 128 + c4 * 4 : 0), ok);
    }
    for (int i = tid; i < DS * 128; i += D_THREADS) {  // 32 rows x 128 float4 of values
      const int r = i >> 7, c4 = i & 127;
      const bool ok = s0 + r < n_live;
      cp_async16(&sm.v[stage][r][c4 * 4], vals + (ok ? (s0 + r) * 512 + c4 * 4 : 0), ok);
    }
    cp_async_commit();
  };
  load_tile(0, t_begin);

  // query tile, divided by sqrt(128) with the IEEE division of the reference (rows past hw are zero)
  const float* qk = p.a.qk + static_cast<int64_t>(query_set(p.a, obj)) * p.a.hw * 128;
  for (int i = tid; i < DQ * 32; i += D_THREADS) {
    const int r = i >> 5, c4 = i & 31;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < p.a.hw) {
      v = *reinterpret_cast<const float4*>(qk + static_cast<int64_t>(q0 + r) * 128 + c4 * 4);
      v.x = v.x / kSqrtCK; v.y = v.y / kSqrtCK; v.z = v.z / kSqrtCK; v.w = v.w / kSqrtCK;
    }
    *reinterpret_cast<float4*>(&sm.q[r][c4 * 4]) = v;
  }

  // softmax role: row sr, columns [8 ss, 8 ss + 8) of the tile (every one of the 4 threads keeps m, l)
  const int sr = tid >> 2, ss = tid & 3;
  float m_run = -INFINITY, l_run = 0.f;
  // S role: rows [16 srt, +16), slots [16 sch, +16) of the tile
  const int srt = warp & 3, sch = warp >> 2;
  // PV role: all 64 rows, value channels [64 warp, +64)
  float o[4][8][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[i][j][e] = 0.f;

  for (int it = 0; it < ntiles; ++it) {
    const int st = it & 1;
    const int64_t tile = t_begin + it;
    cp_async_wait_all();
    __syncthreads();  // tile `it` visible; every warp is done with the previous tile's P, alpha and stage st ^ 1
    if (it + 1 < ntiles) load_tile(st ^ 1, tile + 1);

    // ---- S = (q/sqrt(128)) . key, 3xTF32
    {
      float acc[2][4];
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
      const float* qa = &sm.q[16 * srt + g][t];
#pragma unroll 4
      for (int kk = 0; kk < 16; ++kk) {
        uint32_t ah[4], al[4];
        split_tf32(qa[8 * kk], ah[0], al[0]);
        split_tf32(qa[8 * QSTR + 8 * kk], ah[1], al[1]);
        split_tf32(qa[8 * kk + 4], ah[2], al[2]);
        split_tf32(qa[8 * QSTR + 8 * kk + 4], ah[3], al[3]);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float* kb = &sm.k[st][16 * sch + 8 * j + g][8 * kk + t];
          uint32_t bh0, bl0, bh1, bl1;
          split_tf32(kb[0], bh0, bl0);
          split_tf32(kb[4], bh1, bl1);
          mma_tf32(acc[j], al, bh0, bh1);  // small terms first
          mma_tf32(acc[j], ah, bl0, bl1);
          mma_tf32(acc[j], ah, bh0, bh1);
        }
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int c = 16 * sch + 8 * j + 2 * t;
        *reinterpret_cast<float2*>(&sm.p[16 * srt + g][c]) = make_float2(acc[j][0], acc[j][1]);
        *reinterpret_cast<float2*>(&sm.p[16 * srt + g + 8][c]) = make_float2(acc[j][2], acc[j][3]);
      }
    }
    __syncthreads();

    // ---- online softmax of the tile
    {
      const int ncols = static_cast<int>(n_live - tile * DS < DS ? n_live - tile * DS : DS);
      float s[8];
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s[j] = (8 * ss + j < ncols) ? sm.p[sr][8 * ss + j] : -INFINITY;  // slots past the live count take no part
        mx = fmaxf(mx, s[j]);
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run, mx);
      const float alpha = expf(m_run - m_new);  // 0 on the first tile (m_run = -inf)
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float pj = __uint_as_float(tf32_rna(expf(s[j] - m_new)));
        sm.p[sr][8 * ss + j] = pj;
        sum += pj;
      }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      l_run = l_run * alpha + sum;
      m_run = m_new;
      if (ss == 0) sm.alpha[sr] = alpha;
    }
    __syncthreads();

    // ---- O = alpha * O + P . V  (TF32; P already rounded, V passed as fp32 bits: the MMA reads its TF32 part)
    {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float a0 = sm.alpha[16 * i + g], a1 = sm.alpha[16 * i + g + 8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          o[i][j][0] *= a0; o[i][j][1] *= a0;
          o[i][j][2] *= a1; o[i][j][3] *= a1;
        }
      }
#pragma unroll
      for (int kk = 0; kk < DS / 8; ++kk) {
        uint32_t a[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          a[i][0] = __float_as_uint(sm.p[16 * i + g][8 * kk + t]);
          a[i][1] = __float_as_uint(sm.p[16 * i + g + 8][8 * kk + t]);
          a[i][2] = __float_as_uint(sm.p[16 * i + g][8 * kk + t + 4]);
          a[i][3] = __float_as_uint(sm.p[16 * i + g + 8][8 * kk + t + 4]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint32_t b0 = __float_as_uint(sm.v[st][8 * kk + t][64 * warp + 8 * j + g]);
          const uint32_t b1 = __float_as_uint(sm.v[st][8 * kk + t + 4][64 * warp + 8 * j + g]);
#pragma unroll
          for (int i = 0; i < 4; ++i) mma_tf32(o[i][j], a[i], b0, b1);
        }
      }
    }
  }

  // ---- partials of this chunk
  const int64_t prow = (static_cast<int64_t>(obj) * p.chunks + chunk) * p.a.hw;
  if (ss == 0 && q0 + sr < p.a.hw) p.part_ml[prow + q0 + sr] = make_float2(m_run, l_run);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = q0 + 16 * i + g + 8 * h;
      if (q >= p.a.hw) continue;
      float* dst = p.part_o + (prow + q) * 512 + 64 * warp + 2 * t;
#pragma unroll
      for (int j = 0; j < 8; ++j) *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(o[i][j][2 * h], o[i][j][2 * h + 1]);
    }
  }
}

constexpr int C_WARPS = 8;

__global__ void __launch_bounds__(32 * C_WARPS) memread_dense_combine_kernel(
    const MemreadArgs a, const float* __restrict__ part_o, const float2* __restrict__ part_ml, int chunk_tiles, int chunks) {
  mivos::pdl_prologue();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t lq = static_cast<int64_t>(blockIdx.x) * C_WARPS + warp;  // = obj * hw + q
  const int hw = a.hw;
  if (lq >= static_cast<int64_t>(a.k_objects) * hw) return;
  const int obj = static_cast<int>(lq / hw), q = static_cast<int>(lq - static_cast<int64_t>(obj) * hw);
  const int64_t live_tiles = (live_slots(a, obj) + DS - 1) / DS;
  const int live = static_cast<int>((live_tiles + chunk_tiles - 1) / chunk_tiles);
  const int64_t base = static_cast<int64_t>(obj) * chunks * hw + q;  // chunk c of this query: base + c * hw
  float M = -INFINITY;
  for (int c = 0; c < live; ++c) M = fmaxf(M, part_ml[base + static_cast<int64_t>(c) * hw].x);
  float L = 0.f;
  float4 acc[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c = 0; c < live; ++c) {  // fixed ascending order
    const int64_t r = base + static_cast<int64_t>(c) * hw;
    const float2 ml = part_ml[r];
    const float w = expf(ml.x - M);
    L = fmaf(w, ml.y, L);
    const float4* src = reinterpret_cast<const float4*>(part_o + r * 512);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float4 v = src[lane + 32 * u];
      acc[u].x = fmaf(w, v.x, acc[u].x);
      acc[u].y = fmaf(w, v.y, acc[u].y);
      acc[u].z = fmaf(w, v.z, acc[u].z);
      acc[u].w = fmaf(w, v.w, acc[u].w);
    }
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) acc[u] = make_float4(acc[u].x / L, acc[u].y / L, acc[u].z / L, acc[u].w / L);
  store_read_row(a, obj, q, lane, acc);
}

// Chunk length (tiles of DS slots) as a function of hw alone.  Small frames have few query tiles and need many
// chunks to fill the GPU; large frames fill it with query tiles and must keep the partials (K x chunks x hw x 2 KB)
// bounded.  The length grows with the cube of the query-tile count: 1620 queries (480p at stride 16) get
// 100 tiles = 3200 slots (~2 frames), 3600 queries (720p) 1054 tiles (~9.4 frames); never fewer than 8 tiles.
int dense_chunk_tiles(int hw) {
  const int64_t qt = ceil_div(hw, DQ);
  const int64_t t = ceil_div64(qt * qt * qt, 176);
  return static_cast<int>(t < 8 ? 8 : t);
}

struct DensePlan {
  int chunk_tiles, chunks, qtiles;
  int64_t off_ml, bytes;
};

DensePlan dense_plan(int k_objects, int64_t slots_cap, int hw) {
  DensePlan pl;
  pl.chunk_tiles = dense_chunk_tiles(hw);
  pl.chunks = static_cast<int>(ceil_div64(ceil_div64(slots_cap, DS), pl.chunk_tiles));
  pl.qtiles = ceil_div(hw, DQ);
  const int64_t rows = static_cast<int64_t>(k_objects) * pl.chunks * hw;
  pl.off_ml = rows * 512 * 4;
  pl.bytes = ((pl.off_ml + rows * 8) + 255) & ~255ll;
  return pl;
}

}  // namespace
}  // namespace mivos

using namespace mivos;

extern "C" MIVOS_API int64_t mivos_memory_read_dense_workspace(int k_objects, int64_t slots_cap, int hw) {
  if (k_objects < 1 || k_objects > kMaxObjects || slots_cap < 1 || slots_cap >= (1ll << 31) - 65536 || hw < 1) return -1;
  return dense_plan(k_objects, slots_cap, hw).bytes;
}

namespace {

int memory_read_dense_run(const MemreadArgs& a, void* workspace, int64_t workspace_bytes, cudaStream_t stream) {
  const int64_t slots_cap = a.slots_cap, slots = a.slots;
  const int k_objects = a.k_objects, hw = a.hw;
  MIVOS_REQUIRE(slots_cap >= 1 && slots_cap < (1ll << 31) - 65536 && slots >= 1 && slots <= slots_cap,
                "memory_read_dense: bad slot count %lld (cap %lld)", (long long)slots, (long long)slots_cap);
  MIVOS_REQUIRE(workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0,
                "memory_read_dense: workspace null or not 256-byte aligned");
  const DensePlan pl = dense_plan(k_objects, slots_cap, hw);
  MIVOS_REQUIRE(workspace_bytes >= pl.bytes, "memory_read_dense: workspace %lld < %lld bytes", (long long)workspace_bytes,
                (long long)pl.bytes);
  MIVOS_REQUIRE(pl.chunks <= 65535, "memory_read_dense: %d chunks of the memory axis exceed the grid", pl.chunks);

  static bool configured = false;
  if (!configured) {
    MIVOS_CUDA_OK(cudaFuncSetAttribute(memread_dense_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(sizeof(DenseSmem))));
    configured = true;
  }
  uint8_t* w = static_cast<uint8_t*>(workspace);
  DenseParams p;
  p.a = a;
  p.chunk_tiles = pl.chunk_tiles;
  p.chunks = pl.chunks;
  p.part_o = reinterpret_cast<float*>(w);
  p.part_ml = reinterpret_cast<float2*>(w + pl.off_ml);
  launch_pdl(memread_dense_kernel, dim3(pl.qtiles, pl.chunks, k_objects), D_THREADS, sizeof(DenseSmem), stream, p);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  MIVOS_CUDA_OK(cudaGetLastError());

  launch_pdl(memread_dense_combine_kernel, dim3(ceil_div(k_objects * hw, C_WARPS)), 32 * C_WARPS, 0, stream, a,
             static_cast<const float*>(p.part_o), static_cast<const float2*>(p.part_ml), pl.chunk_tiles, pl.chunks);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  MIVOS_CUDA_OK(cudaGetLastError());
  return MIVOS_OK;
}

}  // namespace

extern "C" MIVOS_API int mivos_memory_read_dense(const float* bank_k, const float* bank_v, int64_t slots_cap,
                                                 int k_objects, int64_t slots, const float* qk, int hw, int q_div,
                                                 void* out, int out_cstride, int out_coff, int out_halo_h,
                                                 int out_halo_w, void* workspace, int64_t workspace_bytes,
                                                 const int32_t* dyn_slots, int out_f16, mivos_stream_t stream_) {
  const MemreadArgs a{bank_k, bank_v, slots_cap, k_objects, slots, dyn_slots, qk, hw, q_div,
                      out, out_cstride, out_coff, out_halo_h, out_halo_w, out_f16, 0};
  const int rc = memread_check_args(a, "memory_read_dense");
  if (rc != MIVOS_OK) return rc;
  return memory_read_dense_run(a, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" MIVOS_API int mivos_memory_read_dense_sets(const float* bank_k, const float* bank_v, int64_t slots_cap,
                                                      int k_objects, int64_t slots, const float* qk, int hw, int sets,
                                                      void* out, int out_cstride, int out_coff, int out_halo_h,
                                                      int out_halo_w, void* workspace, int64_t workspace_bytes,
                                                      const int32_t* dyn_slots, int out_f16, mivos_stream_t stream_) {
  MemreadArgs a{bank_k, bank_v, slots_cap, k_objects, slots, dyn_slots, qk, hw, 0,
                out, out_cstride, out_coff, out_halo_h, out_halo_w, out_f16, 0};
  int rc = memread_sets_args(a, sets, "memory_read_dense_sets");
  if (rc == MIVOS_OK) rc = memread_check_args(a, "memory_read_dense_sets");
  if (rc != MIVOS_OK) return rc;
  return memory_read_dense_run(a, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" MIVOS_API int mivos_memory_read_dense_groups(const float* bank_k, const float* bank_v, int64_t slots_cap,
                                                        int k_objects, int64_t slots, const float* qk, int hw,
                                                        int groups, const int32_t* first, void* out, int out_cstride,
                                                        int out_coff, int out_halo_h, int out_halo_w, void* workspace,
                                                        int64_t workspace_bytes, const int32_t* dyn_slots, int out_f16,
                                                        mivos_stream_t stream_) {
  MemreadArgs a{bank_k, bank_v, slots_cap, k_objects, slots, dyn_slots, qk, hw, 0,
                out, out_cstride, out_coff, out_halo_h, out_halo_w, out_f16, 0};
  int rc = memread_check_args(a, "memory_read_dense_groups");
  if (rc == MIVOS_OK) rc = memread_groups_args(a, groups, first, "memory_read_dense_groups");
  if (rc != MIVOS_OK) return rc;
  return memory_read_dense_run(a, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}
