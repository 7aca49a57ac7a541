// Internal interface between the memory-read translation units (memread.cu, memread_tc.cu).
#pragma once
#include "host_util.h"

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

struct MemreadPlan {
  int algo;
  int qtile;      // queries per CTA
  int slot_tile;  // bank slots per inner tile
  int qtiles;
  int splits;  // CTAs along the memory axis
  int nlists;  // candidate lists per (object, query): splits (exact) or splits * kTcHalves (tensor cores)
  int tiles_per_split;
  int kcap;  // list capacity per (object, query, split)
  // candidate lists are int2 {score bits, slot}: one 8-byte store per append, one load per read
  int64_t off_list, off_cnt, off_flag, bytes;
};

MemreadPlan memread_plan(int k_objects, int64_t slots, int hw, int top_k, int algo);

// First candidate list of a plan inside its workspace.  The tensor-core plan's lists (kTcCandCap * 8 = 4096 bytes
// each) start on a 4 KB boundary, so no list straddles a 4 GB boundary and the generator bumps only the low
// word of its append pointer (the plan reserves the 4 KB of slack).
inline uint8_t* plan_lists(void* ws, const MemreadPlan& pl) {
  uint8_t* p = static_cast<uint8_t*>(ws) + pl.off_list;
  if (pl.algo != MIVOS_MEMREAD_TCGEN05) return p;
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 4095) & ~static_cast<uintptr_t>(4095));
}

// `flags` (optional, [K*hw]): only CTAs owning a flagged query do any work.
int launch_exact_candidates(const float* bank_k, int64_t slots_cap, int k_objects, int64_t slots,
                            const float* qk, int hw, int q_div, int top_k, const MemreadPlan& pl, void* ws,
                            const int* flags, const int* dyn_slots, cudaStream_t stream);
// Lists come from `pl`/`ws` (approximate scores that need the exact re-score when pl.algo is the tensor-core plan).
// `flags` (optional, [K*hw]) and `pass`: pass 0 serves the queries whose flag is clear and SETS the flag of a query
// whose lists hold more in-band candidates than the stage can stage (instead of selecting it); pass 1 serves only
// the flagged queries (from the exact lists of the fallback).  flags == nullptr: one pass over every query.
int launch_select(const float* bank_k, const float* bank_v, int64_t slots_cap, int k_objects,
                  const float* qk, int hw, int q_div, int top_k, const MemreadPlan& pl, void* ws,
                  const MemreadPlan* fb, void* fb_ws, int* flags, int pass, const float* qnorm,
                  const float* kmax2, const int* tau_g, void* out, int out_cstride, int out_coff, int halo_h,
                  int halo_w, int out_f16, int32_t* topk_idx, float* topk_val, cudaStream_t stream);

bool memread_tc_available();
int memread_tc_run(const float* bank_k, const float* bank_v, int64_t slots_cap, int k_objects,
                   int64_t slots, const float* qk, int hw, int q_div, int top_k, void* out, int out_cstride,
                   int out_coff, int halo_h, int halo_w, int out_f16, int32_t* topk_idx, float* topk_val,
                   void* workspace, const int* dyn_slots, cudaStream_t stream);

}  // namespace mivos
