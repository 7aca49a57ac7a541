// Object groups of the *_groups entry points: lock-step clips with different object counts.  A batch of `maps`
// object maps is split into `groups` runs of consecutive maps by a DEVICE table `first` of groups + 1 int32 entries
// (exclusive prefix sums of the groups' object counts): group g owns maps [first[g], first[g+1]).  The table is read
// at run time, so the host cannot check it; a map that no well-formed group holds takes part in nothing.
#pragma once
#include <cuda_runtime.h>

namespace mivos {

// Group of map `i`: the g with first[g] <= i < first[g+1], or -1 when no group holds it.  A group counts only when
// it lies inside [0, maps] and is not empty; a table that is not ascending yields -1 (or a group that does hold `i`),
// never an index outside [0, groups).
__device__ __forceinline__ int map_group(const int* __restrict__ first, int groups, int maps, int i) {
  int lo = 0, hi = groups - 1;  // largest g with first[g] <= i, for an ascending table
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(first + mid) <= i) lo = mid;
    else hi = mid - 1;
  }
  const int a = __ldg(first + lo), b = __ldg(first + lo + 1);
  return (a >= 0 && a <= i && i < b && b <= maps) ? lo : -1;
}

// Maps [*m0, *m0 + *n) of group g, or false when the group is empty or outside [0, maps].
__device__ __forceinline__ bool group_range(const int* __restrict__ first, int maps, int g, int* m0, int* n) {
  const int a = __ldg(first + g), b = __ldg(first + g + 1);
  *m0 = a;
  *n = b - a;
  return a >= 0 && a < b && b <= maps;
}

}  // namespace mivos
