// pass_core.h -- the "fused pass" vocabulary shared by the solver engines added in the section 8(f)
// widening (qmr, lsqr, lsmr, idrs).
//
// An engine is written as a sequence of PASSES over the vectors.  A pass is a small functor
//
//   struct P {
//     static constexpr int NRED = r;          // sums it produces (0 .. kPassMaxRed)
//     bool   skip() const;                    // true once the solver's device-side `done` flag is set
//     void   load();                          // cache the device-resident scalars the element update needs
//     void   elem(int64_t i, double *acc);    // the fused element update of row i; adds into acc[0..r)
//     double *sums() const;                   // where the r totals go (device scalars of the solver)
//     void   finish(const double *tot) const; // the scalar section that follows the reduction
//   };
//
// and a backend runs it:  Backend::pass(P, n).  On the GPU (pass.cuh) that is ONE kernel: a grid of a
// multiple of the SM count streams the rows, reduces the r sums deterministically (fixed slot order,
// last block finishes) and the finishing thread executes finish() -- so every scalar recurrence of
// the solver (Lanczos coefficients, plane rotations, stopping tests, the done flag) stays in device
// memory and the host only polls `done` every few iterations.  On multi-GPU contexts the totals are
// written to sums(), allreduced (NCCL) and finish() runs in a one-thread kernel.
//
// Everything in the *_core.h headers is plain C++ (B200_HD = __host__ __device__ under nvcc, inline
// otherwise), so that tests/hostsim -- TEST INFRASTRUCTURE, never linked into libb200krylov.so -- can run
// the very same functors, scalar sections and driver loops on the CPU with a serial backend and compare
// them with the CPU checker.  The product library instantiates the drivers with the CUDA backend only: there
// is no CPU fallback in it.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "complex.h"

#ifdef __CUDACC__
#define B200_HD __host__ __device__ __forceinline__
#define B200_UNROLL _Pragma("unroll")
#else
#define B200_HD inline
#define B200_UNROLL
#endif

namespace b200 {

constexpr int kPassMaxRed = 16;   // sums per pass (IDR(s) with s <= 16 needs s)

// machine epsilon of the vector element type (eps(real(T)) of the reference's default tolerances)
template <typename T>
B200_HD double eps_of() {
  return sizeof(typename real_of<T>::type) == 8 ? 2.220446049250313e-16 : 1.1920928955078125e-07;
}

// LinearAlgebra.givensAlgorithm(f, g) for real arguments -> (c, s, r) with [c s; -s c][f; g] = [r; 0]
// (same convention as the GMRES / MINRES engines, pinned against the fixtures of reference test/hessenberg.jl by the test-suite)
B200_HD void givens_real(double f, double g, double &c, double &s, double &r) {
  if (g == 0.0) { c = 1.0; s = 0.0; r = f; return; }
  if (f == 0.0) { c = 0.0; s = 1.0; r = g; return; }
  r = hypot(f, g);
  c = f / r;
  s = g / r;
  if (fabs(f) > fabs(g) && c < 0.0) { c = -c; s = -s; r = -r; }
}

// Scalar-only step (no vector traffic): a pass with n == 0 whose finish() takes no totals.
// Engines use it to publish `done` after the last vector pass of an iteration.
template <typename S, void (*FN)(S *)>
struct ScalarStep {
  static constexpr int NRED = 0;
  S *s;
  B200_HD bool skip() const { return false; }
  B200_HD void load() {}
  B200_HD void elem(int64_t, double *) const {}
  B200_HD double *sums() const { return nullptr; }
  B200_HD void finish(const double *) const { FN(s); }
};

}  // namespace b200
