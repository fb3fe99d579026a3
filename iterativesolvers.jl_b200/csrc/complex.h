// complex.h -- the complex element types ComplexF64 / ComplexF32 (B200_CF64 / B200_CF32): cplx<double>, cplx<float>.
//
// Plain C++ (B200_HD = __host__ __device__ under nvcc, inline otherwise) so that the CPU test backend (tests/hostsim)
// compiles the same arithmetic as the device.  Layout: interleaved (re, im), the layout of Julia's Complex{T} and of
// numpy's complex128 / complex64.  The alignment is that of R, NOT 2 sizeof(R): numpy's complex128 and Julia's ComplexF64
// are only 8-byte aligned, so a caller's vector may start 8 bytes off a 16-byte boundary.  Element accesses through
// cplx<R> are therefore always legal; the 16-byte (8-byte) vector accesses of ld_stream / __ldg below are used only where
// a launcher has checked the pointer.
#pragma once
#include <math.h>

#ifndef B200_HD
#ifdef __CUDACC__
#define B200_HD __host__ __device__ __forceinline__
#else
#define B200_HD inline
#endif
#endif

namespace b200 {

template <typename R>
struct cplx {
  R re, im;
  cplx() = default;   // trivial, like double: scratch blocks holding complex scalars stay memset / memcpy-able
  B200_HD constexpr cplx(R r) : re(r), im(0) {}
  B200_HD constexpr cplx(R r, R i) : re(r), im(i) {}
  template <typename Q>
  B200_HD explicit constexpr cplx(const cplx<Q> &o) : re((R)o.re), im((R)o.im) {}
  B200_HD cplx &operator+=(const cplx &o) {
    re = re + o.re;
    im = im + o.im;
    return *this;
  }
  B200_HD cplx &operator-=(const cplx &o) {
    re = re - o.re;
    im = im - o.im;
    return *this;
  }
};
static_assert(sizeof(cplx<double>) == 16 && alignof(cplx<double>) == 8, "ComplexF64 layout");
static_assert(sizeof(cplx<float>) == 8 && alignof(cplx<float>) == 4, "ComplexF32 layout");

template <typename T>
struct is_cplx {
  static constexpr bool value = false;
};
template <typename R>
struct is_cplx<cplx<R>> {
  static constexpr bool value = true;
};
// the real component type: R for cplx<R>, T itself for real T
template <typename T>
struct real_of {
  typedef T type;
};
template <typename R>
struct real_of<cplx<R>> {
  typedef R type;
};

template <typename R>
B200_HD cplx<R> operator+(const cplx<R> &a, const cplx<R> &b) { return cplx<R>(a.re + b.re, a.im + b.im); }
template <typename R>
B200_HD cplx<R> operator-(const cplx<R> &a, const cplx<R> &b) { return cplx<R>(a.re - b.re, a.im - b.im); }
template <typename R>
B200_HD cplx<R> operator-(const cplx<R> &a) { return cplx<R>(-a.re, -a.im); }
// Products and sums of the complex product rounded one by one (no fused multiply-add), in device code as on the host
// (tests/hostsim builds with -ffp-contract=off): the compiler's contraction choices may differ between two instantiations
// of one kernel (the SpMV's vector- and scalar-load forms), which would make their results differ in the last bit.
#ifdef __CUDA_ARCH__
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
#else
template <typename R>
inline R mul_rn(R a, R b) { return a * b; }
template <typename R>
inline R add_rn(R a, R b) { return a + b; }
template <typename R>
inline R sub_rn(R a, R b) { return a - b; }
#endif
template <typename R>
B200_HD cplx<R> operator*(const cplx<R> &a, const cplx<R> &b) {
  return cplx<R>(sub_rn(mul_rn(a.re, b.re), mul_rn(a.im, b.im)), add_rn(mul_rn(a.re, b.im), mul_rn(a.im, b.re)));
}
template <typename R>
B200_HD cplx<R> operator*(R a, const cplx<R> &b) { return cplx<R>(a * b.re, a * b.im); }
template <typename R>
B200_HD cplx<R> conj(const cplx<R> &a) { return cplx<R>(a.re, -a.im); }
template <typename R>
B200_HD R abs2(const cplx<R> &a) { return a.re * a.re + a.im * a.im; }

// Scaled (Smith) division: no overflow / underflow of c^2 + d^2 for large or small denominators.  Dividing by a value with a
// zero imaginary part is exact (the scale factor is 0): (a + i b) / (c + 0 i) = a / c + i b / c.
template <typename R>
B200_HD cplx<R> operator/(const cplx<R> &x, const cplx<R> &y) {
  const R a = x.re, b = x.im, c = y.re, d = y.im;
  if (fabs(c) >= fabs(d)) {
    const R r = d / c, den = c + d * r;
    return cplx<R>((a + b * r) / den, (b - a * r) / den);
  }
  const R r = c / d, den = c * r + d;
  return cplx<R>((a * r + b) / den, (b * r - a) / den);
}

}  // namespace b200

#ifdef __CUDACC__
// A complex value across the lanes of a warp: two shuffles.
template <typename R>
__device__ __forceinline__ b200::cplx<R> __shfl_xor_sync(unsigned mask, b200::cplx<R> v, int lane_mask, int width = 32) {
  return b200::cplx<R>(__shfl_xor_sync(mask, v.re, lane_mask, width), __shfl_xor_sync(mask, v.im, lane_mask, width));
}
// One 16-byte (ComplexF64) / 8-byte (ComplexF32) read-only load: p must be aligned to 2 sizeof(R).
__device__ __forceinline__ b200::cplx<double> __ldg(const b200::cplx<double> *p) {
  const double2 v = __ldg(reinterpret_cast<const double2 *>(p));
  return b200::cplx<double>(v.x, v.y);
}
__device__ __forceinline__ b200::cplx<float> __ldg(const b200::cplx<float> *p) {
  const float2 v = __ldg(reinterpret_cast<const float2 *>(p));
  return b200::cplx<float>(v.x, v.y);
}
#endif
