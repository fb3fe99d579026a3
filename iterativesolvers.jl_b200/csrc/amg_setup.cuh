// amg_setup.cuh -- the device setup of smoothed aggregation (amg_setup.cu) as amg.cu sees it.
#pragma once
#include <vector>

#include "amg_core.h"
#include "csr.cuh"

namespace b200 {

struct AmgDevLevel {
  const b200_csr *A = nullptr;   // level 0: the caller's operator; coarser levels: owned
  b200_csr *P = nullptr, *R = nullptr;
  int64_t n = 0;
  void *w = nullptr, *b = nullptr, *x = nullptr, *u0 = nullptr, *u1 = nullptr, *inv = nullptr;
  std::vector<int> agg;
  int pass1_launches = 0;   // launches of pass 1 in this level's aggregation (0 on the coarsest level)
};

// Builds the hierarchy of A (element type T, int32 row offsets, single GPU) on the device: every level's A (level 0 is
// A itself), P, the smoother weights w, the aggregates (host copy) and the coarsest level's inverse, each equal bit for
// bit to amg_setup's levels rounded to T.  levels is filled as it goes (the caller frees it on failure too).
// seconds: input checks, aggregation, P, RAP + coarse inverse, level operators.
template <typename T>
int amg_device_setup(b200_ctx *ctx, const b200_csr *A, const AmgOptions &o, std::vector<AmgDevLevel> *levels,
                     std::vector<int64_t> *nnz_P, double *seconds);

}  // namespace b200
