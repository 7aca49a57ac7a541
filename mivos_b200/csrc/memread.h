// Internal interface between the memory-read translation units (memread.cu, memread_tc.cu, memread_dense.cu,
// memread_wide.cu):
// the operands of a read, the workspace layout of the top-k read, and the device pieces the kernels share.
#pragma once
#include "groups.cuh"
#include "host_util.h"

#include <cuda_fp16.h>
#include <cstdint>

namespace mivos {

constexpr int kMaxSplits = 16;
constexpr int kMaxObjects = 256;  // objects (x lock-step clips) one memory-read call may serve
constexpr int kTcCandCap = 512;   // candidates one (query, split) may hold while streaming (tensor-core path)
// A list ends at most kTcCandCap - 128 long (the streaming invariant: it is compacted against the current threshold
// whenever it passes that, and flagged for the exact fallback if that does not help).  There is no further per-list
// cap at the end of the kernel — with a fixed cap of 224 and top-k 50 about 5 % of the
// queries ended above it, and ONE flagged query costs the exact fallback a whole 32-query tile over every slot
// (5.1 ms per read).  The decision now belongs to the selection stage (pass A), which sees all lists of a query.
constexpr int kSelMaxSurvivors = 1024;   // candidates (staged) / survivors (re-scored) the selection stage holds per query
constexpr int kTcHalves = 2;      // column halves of a slot tile, one thread (and list) per query each
constexpr int kMaxLists = kMaxSplits * kTcHalves;  // candidate lists per (object, query)
// margin = 2*eps, eps = 1.05 * 2^-9 * ||q/sqrt(128)|| * max||key||  (see memread_tc.cu)
constexpr float kTcMarginFactor = 2.0f * 1.05f * 0.001953125f;
constexpr float kSqrtCK = 11.313708498984761f;  // sqrt(128) rounded to fp32, as the reference's divisor

// Operands of one read (top-k or dense), as the C entry points receive them.
struct MemreadArgs {
  // bank: keys [k_objects, slots_cap, 128], values [k_objects, slots_cap, 512]; the first `slots` rows are live, or
  // *dyn_slots of them when that optional device scalar is given (CUDA-graph replay)
  const float* bank_k;
  const float* bank_v;
  int64_t slots_cap;
  int k_objects;
  int64_t slots;
  const int* dyn_slots;
  // queries [sets, hw, 128]; object o reads set o / q_div (q_div 0: one set for all objects)
  const float* qk;
  int hw, q_div;
  // output window: 512 channels at out_coff of rows out_cstride wide; HALO rows when halo_w > 0, else row = obj * hw + q
  void* out;
  int out_cstride, out_coff, halo_h, halo_w, out_f16;
  // per-set counts (the *_sets entry points): query set s reads dyn_slots[s * dyn_set_stride]; 0: one count for all
  int dyn_set_stride;
  // object groups (the *_groups entry points): object o reads query set g and count dyn_slots[g] of the group g that
  // holds it (groups.cuh, `groups` + 1 device entries); null: the q_div / stride mapping above
  const int* first;
  int groups;
};

// The operand checks both entry points share; `who` prefixes the error text.  MIVOS_OK or MIVOS_ERR_INVALID.
int memread_check_args(const MemreadArgs& a, const char* who);
// The per-set form's extra checks (counts given, `sets` divides the objects); sets q_div = objects per set and the
// count stride.  MIVOS_OK or MIVOS_ERR_INVALID.
int memread_sets_args(MemreadArgs& a, int sets, const char* who);
// The grouped form's extra checks (counts and table given, 1 <= groups <= objects); sets the group table and the
// count stride.  MIVOS_OK or MIVOS_ERR_INVALID.
int memread_groups_args(MemreadArgs& a, int groups, const int* first, const char* who);

struct MemreadPlan {
  int algo;
  int qtiles;
  int splits;  // CTAs along the memory axis
  int nlists;  // candidate lists per (object, query): splits (exact) or splits * kTcHalves (tensor cores)
  int tiles_per_split;
  int kcap;  // list capacity per (object, query, split)
  // candidate lists (int2 {score bits, slot}: one 8-byte store per append, one load per read) start the plan's
  // workspace, their lengths follow at off_cnt
  int64_t off_cnt, bytes;
};

MemreadPlan memread_plan(int k_objects, int64_t slots, int hw, int top_k, int algo);

// First candidate list of a plan inside its workspace.  The tensor-core plan's lists (kTcCandCap * 8 = 4096 bytes
// each) start on a 4 KB boundary, so no list straddles a 4 GB boundary and the generator bumps only the low
// word of its append pointer (the plan reserves the 4 KB of slack).
inline uint8_t* plan_lists(void* ws, const MemreadPlan& pl) {
  uint8_t* p = static_cast<uint8_t*>(ws);
  if (pl.algo != MIVOS_MEMREAD_TCGEN05) return p;
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 4095) & ~static_cast<uintptr_t>(4095));
}

// Workspace of the top-k read (byte offsets): the tensor-core plan | the exact plan (fallback) | overflow flags
// [K*hw] | key-norm maxima [kMaxObjects] | scaled queries [K*hw*128] (one set per object at most; 16-byte aligned:
// TMA source, float4 stores) | their norms [K*hw] | shared thresholds [K*hw].  The [K*hw] arrays are padded to 256
// bytes; flags and maxima are adjacent so that one memset clears both.
struct MemreadWorkspace {
  MemreadPlan tc, ex;
  int64_t off_ex, off_overflow, off_kmax2, off_qs, off_qnorm, off_tau, bytes;
};

MemreadWorkspace memread_workspace(int k_objects, int64_t slots, int hw, int top_k);

// `flags` (optional, [K*hw]): only CTAs owning a flagged query do any work.
int launch_exact_candidates(const MemreadArgs& a, int top_k, const MemreadPlan& pl, void* ws, const int* flags,
                            cudaStream_t stream);
// Lists come from `pl`/`ws` (approximate scores that need the exact re-score when pl.algo is the tensor-core plan).
// `flags` (optional, [K*hw]) and `pass`: pass 0 serves the queries whose flag is clear and SETS the flag of a query
// whose lists hold more in-band candidates than the stage can stage (instead of selecting it); pass 1 serves only
// the flagged queries (from the exact lists of the fallback).  flags == nullptr: one pass over every query.
int launch_select(const MemreadArgs& a, int top_k, const MemreadPlan& pl, void* ws, int* flags, int pass,
                  const float* qnorm, const float* kmax2, const int* tau_g, int32_t* topk_idx, float* topk_val,
                  cudaStream_t stream);

int memread_tc_run(const MemreadArgs& a, int top_k, int32_t* topk_idx, float* topk_val, void* workspace,
                   cudaStream_t stream);

// float <-> int with the same ordering (so atomicMax on the int is a max on the float)
__device__ __forceinline__ int float_ordered(float f) {
  const int b = __float_as_int(f);
  return b >= 0 ? b : b ^ 0x7fffffff;
}
__device__ __forceinline__ float ordered_float(int o) { return __int_as_float(o >= 0 ? o : o ^ 0x7fffffff); }

// Live bank slots of query set `set`: the device-side count when there is one (dyn_slots[set * set_stride]; stride 0:
// one count for every set), never more than the capacity (the count indexes the bank).
__device__ __forceinline__ int64_t live_slots(const int* dyn_slots, int64_t slots, int64_t slots_cap, int set = 0,
                                              int set_stride = 0) {
  const int64_t n = dyn_slots ? static_cast<int64_t>(dyn_slots[set * set_stride]) : slots;
  return n < slots_cap ? n : slots_cap;
}
// Query set of object `obj` and its live slots.  An object in no group (a malformed group table) reads query set 0
// over no live slot: it takes part in no other object's read and reads no bank slot.
__device__ __forceinline__ int object_group(const MemreadArgs& a, int obj) {
  if (a.first) return map_group(a.first, a.groups, a.k_objects, obj);
  return a.q_div > 0 ? obj / a.q_div : 0;
}
__device__ __forceinline__ int query_set(const MemreadArgs& a, int obj) {
  const int g = object_group(a, obj);
  return g < 0 ? 0 : g;
}
__device__ __forceinline__ int64_t live_slots(const MemreadArgs& a, int obj) {
  const int g = object_group(a, obj);
  return g < 0 ? 0 : live_slots(a.dyn_slots, a.slots, a.slots_cap, g, a.dyn_set_stride);
}

// The exact score of one key row against a scaled query (q / sqrt(128)): fmaf in ascending channel order.  Every
// read that selects slots ranks them by this value.  The chain starts at +0, so it never yields -0.
__device__ __forceinline__ float exact_score(const float* __restrict__ key, const float* qs) {
  float acc = 0.f;
#pragma unroll 16
  for (int c4 = 0; c4 < 32; ++c4) {
    const float4 kv = *reinterpret_cast<const float4*>(key + c4 * 4);
    acc = fmaf(kv.x, qs[c4 * 4 + 0], acc);
    acc = fmaf(kv.y, qs[c4 * 4 + 1], acc);
    acc = fmaf(kv.z, qs[c4 * 4 + 2], acc);
    acc = fmaf(kv.w, qs[c4 * 4 + 3], acc);
  }
  return acc;
}

// Output row of (object, query) and the store of its 512 read-out channels by one warp: the lane holds the float4
// pieces lane, lane + 32, lane + 64, lane + 96.
__device__ __forceinline__ void store_read_row(const MemreadArgs& a, int obj, int q, int lane, const float4 (&v)[4]) {
  int64_t row;
  if (a.halo_w > 0) {
    const int y = q / a.halo_w, x = q - y * a.halo_w;
    row = (static_cast<int64_t>(obj) * (a.halo_h + 2) + y + 1) * (a.halo_w + 2) + x + 1;
  } else {
    row = static_cast<int64_t>(obj) * a.hw + q;
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int c = (lane + 32 * u) * 4;
    if (a.out_f16) {
      const __half2 h01 = __floats2half2_rn(v[u].x, v[u].y), h23 = __floats2half2_rn(v[u].z, v[u].w);
      uint2 pk;
      pk.x = *reinterpret_cast<const uint32_t*>(&h01);
      pk.y = *reinterpret_cast<const uint32_t*>(&h23);
      *reinterpret_cast<uint2*>(static_cast<__half*>(a.out) + row * a.out_cstride + a.out_coff + c) = pk;
    } else {
      *reinterpret_cast<float4*>(static_cast<float*>(a.out) + row * a.out_cstride + a.out_coff + c) = v[u];
    }
  }
}

}  // namespace mivos
