// obstacle_ids.cuh — which slot's warm start a slot takes when the obstacle selection moves obstacles between slots
// (rda_set_obstacle_ids, DESIGN.md §7.4).
//
// prev [N] are the ids the slots carried in the last solve, cur [N] the ids they carry in the next one.  The k-th slot
// (in slot order) carrying id X takes the state of the k-th slot that carried X, so the padding copies of a repeated
// last obstacle match copy to copy.  An id below 0 is "no obstacle" and never matches; a slot without a match gets -1
// (the caller writes the cold-start values there).
//
// A plain function compiled by nvcc for k_remap_slots (rda_kernels.cu) and by g++ for the CPU twin
// (tests/cpu_twin/obstacle_ids.cpp), O(N) per slot.
#pragma once
#include "rda_hd.h"

namespace rda {

RDA_HD int obstacle_slot_source(const int* prev, const int* cur, int N, int n) {
  const int id = cur[n];
  if (id < 0) return -1;
  int k = 0;                                           // copies of id before slot n
  for (int i = 0; i < n; ++i) k += cur[i] == id;
  for (int i = 0; i < N; ++i)
    if (prev[i] == id && k-- == 0) return i;
  return -1;
}

}  // namespace rda
