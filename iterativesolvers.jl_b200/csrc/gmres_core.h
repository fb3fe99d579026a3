// gmres_core.h -- gmres!(x, A, b; Pl, Pr, abstol, reltol, restart, maxiter, initially_zero, orth_meth) of reference
// src/gmres.jl:184-222 (iterate :57-106, update_residual! :224-233, init! :235-255, solve_least_squares! :262-271,
// update_solution! :273-283, expand! :285-304; orthogonalize_and_normalize! src/orthogonalize.jl:13-79; FastHessenberg
// ldiv! src/hessenberg.jl:15-46) written as fused passes (pass_core.h) for GENERAL operators and preconditioners:
// A, Pl and Pr may be device callbacks (`b200_linop`: the reference's duck-typed `mul!(y, A, x)` / `ldiv!(y, P, x)`
// contract, docs/src/getting_started.md:25-30, docs/src/preconditioning.md:5-15) or Jacobi diagonals.  For a
// `b200_csr` operator with Identity / Jacobi the engine of gmres.cu (register-blocked Gram-Schmidt kernels with 128-bit
// accesses) is the fast path; this one has the same structure with every scalar of the recurrence -- the Hessenberg
// matrix, the null-vector residual recurrence, the Givens least-squares solve -- in device memory: the host reads one
// flag word per inner iteration (restart? converged?).
//
//   expand!      next = Pl \ (A (Pr \ V[:, k]))            callbacks / SpMV / Jacobi passes                  :285-304
//   MGS          k passes (w -= h[i-1] v[i-1] fused with h[i] = <v[i], w>) + 1 (last update + ||w||^2)      orth :67-79
//   CGS          ceil(k/16) dot passes (16 sums each) + ceil(k/16) update passes (the last one with ||w||^2)     :41-51
//   DGKS         CGS + re-orthogonalisation rounds while ||w|| < ||h|| / sqrt(2) (flag read by the host)         :13-39
//   scale        w *= inv(nrm)                                                                                   :36
//   step         H[:, k] ; nullvec recurrence ; residual ; at the end of a cycle the Givens LS solve            :224-233, :262-271
//   update       x += V[:, 1:k-1] y  (through Pr when given)                                                     :273-283
//
// Complex element types (T = cplx<R>): the scalar block is GmScalC, where H, h, corr, nullvec and rhs are complex (fp64
// for ComplexF32 too); every dot is Julia's dot(x, y) = sum conj(x_i) y_i and takes two of a pass's sums, so a CGS / DGKS
// dot pass covers 8 basis columns instead of 16; norms and the DGKS projection sizes use abs2; the least-squares solve
// uses the complex givensAlgorithm with the -conj(s) rotations of src/hessenberg.jl:32,38.  The real instantiations are
// the code they were before complex types existed (if constexpr, overloads on the scalar block).
#pragma once
#include <memory>

#include "complex.h"
#include "pass_core.h"

namespace b200 {

constexpr int kGmMaxRestart = 64;
constexpr int kGmLdh = kGmMaxRestart + 1;
constexpr int kGmBlock = 16;          // basis vectors per dot / update pass

enum { GM_ORTH_MGS = 0, GM_ORTH_CGS = 1, GM_ORTH_DGKS = 2 };     // B200_ORTH_* of the C ABI
enum { GM_FIN = 1, GM_REINIT = 2, GM_DONE = 4, GM_BREAKDOWN = 8 };

struct GmScal {
  double H[kGmLdh * kGmMaxRestart];   // ArnoldiDecomp.H, column-major (restart+1) x restart with leading dimension kGmLdh :14
  double nullvec[kGmLdh];             // Residual.nullvec :27
  double rhs[kGmLdh];                 // after the least-squares solve: y = rhs[0 .. m)
  double h[kGmMaxRestart], corr[kGmMaxRestart];
  double accumulator, current, beta_res, beta, tol, abstol, reltol;
  double nrm2, nrm, proj;
  double sum[kPassMaxRed];
  double *hist;
  long long hist_cap, n_hist, iteration, maxiter;
  int k, restart, m, flags, first, reorth, pad0, pad1;
};

struct GmScalC {                      // GmScal of the complex element types
  cplx<double> H[kGmLdh * kGmMaxRestart];
  cplx<double> nullvec[kGmLdh];
  cplx<double> rhs[kGmLdh];
  cplx<double> h[kGmMaxRestart], corr[kGmMaxRestart];
  double accumulator, current, beta_res, beta, tol, abstol, reltol;
  double nrm2, nrm, proj;
  double sum[kPassMaxRed];
  double *hist;
  long long hist_cap, n_hist, iteration, maxiter;
  int k, restart, m, flags, first, reorth, pad0, pad1;
};
template <typename T>
struct gm_scal {
  typedef GmScal type;
};
template <typename R>
struct gm_scal<cplx<R>> {
  typedef GmScalC type;
};
// basis columns per dot pass: one sum per column, two (re, im) for complex T
template <typename T>
constexpr int gm_dot_block() { return is_cplx<T>::value ? kGmBlock / 2 : kGmBlock; }

template <typename Q>
B200_HD bool gm_done(const Q *q, long long it) { return it >= q->maxiter || q->current <= q->tol; }   // done :55

// after the norm of the (preconditioned) residual is known: init! :252 and what follows it at :126-133 / :96-99
template <typename Q>
B200_HD void gm_set_beta(Q *q, double sumsq) {
  const double beta = sqrt(sumsq);
  q->beta = beta;                               // g.beta :133 / :96
  q->accumulator = 1.0;                         // init_residual! :257-260
  q->beta_res = beta;
  if (q->first) {
    q->current = beta;                          // :126
    q->tol = fmax(q->reltol * beta, q->abstol); // :129
    q->first = 0;
    q->flags = gm_done(q, q->iteration) ? GM_DONE : 0;
    if (!(beta == beta)) q->flags |= GM_DONE | GM_BREAKDOWN;
  }
}

// ---- init!: out = (b - ax) [./ d]; ||out||^2     :241-252
template <typename T>
struct GmResidual {
  static constexpr int NRED = 1;
  const T *b, *ax, *diag;      // ax: A*x or nullptr (initially_zero); diag: Jacobi Pl or nullptr
  T *out;
  typename gm_scal<T>::type *s;
  int is_beta;                 // the norm of this pass is beta (no callback preconditioner follows)
  B200_HD bool skip() const { return false; }
  B200_HD void load() {}
  B200_HD void elem(int64_t i, double *acc) const {
    T r = b[i];                                  // copyto!(first_col, b) :241
    if (ax) r = r - ax[i];                       // first_col .-= Ax :246
    if (diag) r = r / diag[i];                   // ldiv!(Pl, first_col) :249
    out[i] = r;
    if constexpr (is_cplx<T>::value) acc[0] += (double)r.re * (double)r.re + (double)r.im * (double)r.im;
    else acc[0] += (double)r * (double)r;
  }
  B200_HD double *sums() const { return s->sum; }
  B200_HD void finish(const double *tot) const {
    if (is_beta) gm_set_beta(s, tot[0]);
  }
};

template <typename T>
struct GmNorm {                // norm(first_col) after a callback preconditioner :252
  static constexpr int NRED = 1;
  const T *v;
  typename gm_scal<T>::type *s;
  B200_HD bool skip() const { return false; }
  B200_HD void load() {}
  B200_HD void elem(int64_t i, double *acc) const {
    if constexpr (is_cplx<T>::value) acc[0] += (double)v[i].re * (double)v[i].re + (double)v[i].im * (double)v[i].im;
    else acc[0] += (double)v[i] * (double)v[i];
  }
  B200_HD double *sums() const { return s->sum; }
  B200_HD void finish(const double *tot) const { gm_set_beta(s, tot[0]); }
};

// ---- v .*= inv(*src)     :253, orthogonalize.jl:36/:48/:76
template <typename T>
struct GmScale {
  static constexpr int NRED = 0;
  T *v;
  const double *src;
  T inv;
  B200_HD bool skip() const { return false; }
  B200_HD void load() { inv = (T)1 / (T)(*src); }
  B200_HD void elem(int64_t i, double *) const { v[i] = v[i] * inv; }
  B200_HD double *sums() const { return nullptr; }
  B200_HD void finish(const double *) const {}
};

// ---- out = in ./ d   (Jacobi ldiv!; in may alias out)
template <typename T>
struct GmJacobi {
  static constexpr int NRED = 0;
  const T *in, *d;
  T *out;
  B200_HD bool skip() const { return false; }
  B200_HD void load() {}
  B200_HD void elem(int64_t i, double *) const { out[i] = in[i] / d[i]; }
  B200_HD double *sums() const { return nullptr; }
  B200_HD void finish(const double *) const {}
};

// ---- out += in   (x .+= Ax :282)
template <typename T>
struct GmAdd {
  static constexpr int NRED = 0;
  const T *in;
  T *out;
  B200_HD bool skip() const { return false; }
  B200_HD void load() {}
  B200_HD void elem(int64_t i, double *) const { out[i] = out[i] + in[i]; }
  B200_HD double *sums() const { return nullptr; }
  B200_HD void finish(const double *) const {}
};

// ---- modified Gram-Schmidt, orthogonalize.jl:67-79, one pass per basis vector: the update with the previous
// coefficient and the next dot product share the read of w.
template <typename T>
struct GmMgs {
  static constexpr int NRED = is_cplx<T>::value ? 2 : 1;
  const T *vprev, *vi;         // vprev: column whose projection is removed now (nullptr on the first pass);
  T *w;                        // vi: column of the next dot (nullptr on the last pass: ||w||^2 instead)
  typename gm_scal<T>::type *s;
  int iprev, icur;
  T hprev;
  B200_HD bool skip() const { return false; }
  B200_HD void load() { hprev = vprev ? (T)s->h[iprev] : (T)0; }
  B200_HD void elem(int64_t i, double *acc) const {
    T wi = w[i];
    if (vprev) {
      wi = wi - hprev * vprev[i];                // w .-= h[i] .* column :72
      w[i] = wi;
    }
    if constexpr (is_cplx<T>::value) {
      if (vi) {                                  // h[i] = dot(column, w) = sum conj(column) w :71
        const T v = vi[i];
        acc[0] += (double)v.re * (double)wi.re + (double)v.im * (double)wi.im;
        acc[1] += (double)v.re * (double)wi.im - (double)v.im * (double)wi.re;
      } else {
        acc[0] += (double)wi.re * (double)wi.re + (double)wi.im * (double)wi.im;   // nrm = norm(w) :75
      }
    } else {
      acc[0] += vi ? (double)vi[i] * (double)wi    // h[i] = dot(column, w) :71
                   : (double)wi * (double)wi;      // nrm = norm(w) :75
    }
  }
  B200_HD double *sums() const { return s->sum; }
  B200_HD void finish(const double *tot) const {
    if (vi) {
      if constexpr (is_cplx<T>::value) s->h[icur] = cplx<double>(tot[0], tot[1]);
      else s->h[icur] = tot[0];
    } else {
      s->nrm2 = tot[0];
      s->nrm = sqrt(tot[0]);
    }
  }
};

// ---- dst[j0 + j] = <V[:, j0 + j], w>, j < cnt <= 16     mul!(h, V', w) :15 / :43 ; correction :27
template <typename T>
struct GmDots {
  static constexpr int NRED = kGmBlock;
  const T *V;                  // first column of the chunk
  int64_t ld;
  int cnt, j0, to_corr;         // cnt <= gm_dot_block<T>()
  const T *w;
  typename gm_scal<T>::type *s;
  B200_HD bool skip() const { return false; }
  B200_HD void load() {}
  B200_HD void elem(int64_t i, double *acc) const {
    if constexpr (is_cplx<T>::value) {           // sum conj(V[:, j]) w: (re, im) in acc[2j], acc[2j+1]
      const T wv = w[i];
      B200_UNROLL
      for (int j = 0; j < kGmBlock / 2; ++j)
        if (j < cnt) {
          const T v = V[i + j * ld];
          acc[2 * j] += (double)v.re * (double)wv.re + (double)v.im * (double)wv.im;
          acc[2 * j + 1] += (double)v.re * (double)wv.im - (double)v.im * (double)wv.re;
        }
    } else {
      const double wv = (double)w[i];
      B200_UNROLL
      for (int j = 0; j < kGmBlock; ++j)
        if (j < cnt) acc[j] += (double)V[i + j * ld] * wv;
    }
  }
  B200_HD double *sums() const { return s->sum; }
  B200_HD void finish(const double *tot) const {
    auto *dst = to_corr ? s->corr : s->h;
    if constexpr (is_cplx<T>::value) {
      for (int j = 0; j < cnt; ++j) dst[j0 + j] = cplx<double>(tot[2 * j], tot[2 * j + 1]);
    } else {
      for (int j = 0; j < cnt; ++j) dst[j0 + j] = tot[j];
    }
  }
};

// ---- w += sign * V[:, j0 : j0 + cnt] * coef[j0 : j0 + cnt]  (coef in device memory), optionally ||w||^2
//      mul!(w, V, h, -1, 1) :16 / :44 ; w -= V correction :30 ; x += V y :275
enum { GM_COEF_H = 0, GM_COEF_CORR = 1, GM_COEF_Y = 2 };
template <typename T, bool NORM>
struct GmUpdate {
  static constexpr int NRED = NORM ? 1 : 0;
  const T *V;
  int64_t ld;
  int cnt, j0, which;
  double sign;
  T *w;
  typename gm_scal<T>::type *s;
  T c[kGmBlock];
  B200_HD bool skip() const { return false; }
  B200_HD void load() {
    const auto *src = which == GM_COEF_H ? s->h : (which == GM_COEF_CORR ? s->corr : s->rhs);
    B200_UNROLL
    for (int j = 0; j < kGmBlock; ++j) c[j] = j < cnt ? (T)(sign * src[j0 + j]) : (T)0;
  }
  B200_HD void elem(int64_t i, double *acc) const {
    T t = (T)0;
    B200_UNROLL
    for (int j = 0; j < kGmBlock; ++j)
      if (j < cnt) t = t + V[i + j * ld] * c[j];
    const T wi = w[i] + t;
    w[i] = wi;
    if constexpr (is_cplx<T>::value) {
      if (NORM) acc[0] += (double)wi.re * (double)wi.re + (double)wi.im * (double)wi.im;
    } else {
      if (NORM) acc[0] += (double)wi * (double)wi;
    }
  }
  B200_HD double *sums() const { return s->sum; }
  B200_HD void finish(const double *tot) const {
    if (NORM) {
      s->nrm2 = tot[0];
      s->nrm = sqrt(tot[0]);
    }
  }
};

// ---- DGKS: projection_size and the loop condition, orthogonalize.jl:20-33
B200_HD void gm_dgks_first(GmScal *q) {
  double p = 0.0;
  for (int j = 0; j < q->k; ++j) p += q->h[j] * q->h[j];
  q->proj = sqrt(p);                                             // projection_size = norm(h) :22
  q->reorth = q->nrm < (1.0 / sqrt(2.0)) * q->proj;              // :26
}
B200_HD void gm_dgks_next(GmScal *q) {
  double p = 0.0;
  for (int j = 0; j < q->k; ++j) {
    p += q->corr[j] * q->corr[j];
    q->h[j] += q->corr[j];                                       // h .+= correction :31
  }
  q->proj = sqrt(p);                                             // :28
  q->reorth = q->nrm < (1.0 / sqrt(2.0)) * q->proj;
}

// ---- the scalar part of an inner iteration, src/gmres.jl:68-104
B200_HD void gm_step(GmScal *q) {
  const int k = q->k, col = k - 1;
  double *Hc = q->H + (size_t)col * kGmLdh;
  for (int j = 0; j < k; ++j) Hc[j] = q->h[j];                   // H[1:k, k] :68-73
  Hc[k] = q->nrm;                                                // H[k+1, k] = orthogonalize_and_normalize!(...)
  if (q->nrm == 0.0) {                                           // update_residual! :224-233
    q->current = 0.0;
  } else {
    double d = 0.0;
    for (int j = 0; j < k; ++j) d += q->nullvec[j] * Hc[j];
    q->nullvec[k] = -(d / q->nrm);
    q->accumulator += q->nullvec[k] * q->nullvec[k];
    q->current = q->beta_res / sqrt(q->accumulator);
  }
  int flags = 0;
  const int k1 = k + 1;                                          // :78
  q->k = k1;
  if (k1 == q->restart + 1 || gm_done(q, q->iteration + 1)) {    // :82
    // solve_least_squares! :262-271 -- ldiv!(FastHessenberg(H[1:k, 1:k-1]), rhs), src/hessenberg.jl:15-46
    const int m = k1 - 1;
    for (int i = 0; i <= m; ++i) q->rhs[i] = 0.0;
    q->rhs[0] = q->beta;                                         // :265
    double *H = q->H;
    for (int i = 0; i < m; ++i) {                                // hessenberg.jl:24
      double c, s, r;
      givens_real(H[i + i * kGmLdh], H[i + 1 + i * kGmLdh], c, s, r);
      H[i + i * kGmLdh] = c * H[i + i * kGmLdh] + s * H[i + 1 + i * kGmLdh];          // :28
      for (int j = i + 1; j < m; ++j) {                          // :31-35
        const double a = H[i + j * kGmLdh], b = H[i + 1 + j * kGmLdh];
        H[i + j * kGmLdh] = c * a + s * b;
        H[i + 1 + j * kGmLdh] = -s * a + c * b;
      }
      const double a = q->rhs[i], b = q->rhs[i + 1];             // :38-40
      q->rhs[i] = c * a + s * b;
      q->rhs[i + 1] = -s * a + c * b;
    }
    for (int i = m - 1; i >= 0; --i) {                           // UpperTriangular solve :44-45
      double acc = q->rhs[i];
      for (int j = i + 1; j < m; ++j) acc -= H[i + j * kGmLdh] * q->rhs[j];
      q->rhs[i] = acc / H[i + i * kGmLdh];
    }
    q->m = m;
    q->k = 1;                                                    // :90
    flags |= GM_FIN;
    if (!gm_done(q, q->iteration)) flags |= GM_REINIT;           // :93 (sic: the old iteration count)
  }
  q->iteration += 1;
  if (q->hist && q->n_hist < q->hist_cap) q->hist[q->n_hist] = q->current;   // push!(history, :resnorm, ...) :211
  q->n_hist += 1;
  if (gm_done(q, q->iteration)) flags |= GM_DONE;                // :59
  if (!(q->current == q->current)) flags |= GM_DONE | GM_BREAKDOWN;
  q->flags = flags;
}

// ---- complex forms of the scalar sections above (GmScalC)
B200_HD void gm_dgks_first(GmScalC *q) {
  double p = 0.0;
  for (int j = 0; j < q->k; ++j) p += abs2(q->h[j]);
  q->proj = sqrt(p);                                             // projection_size = norm(h) :22
  q->reorth = q->nrm < (1.0 / sqrt(2.0)) * q->proj;              // :26
}
B200_HD void gm_dgks_next(GmScalC *q) {
  double p = 0.0;
  for (int j = 0; j < q->k; ++j) {
    p += abs2(q->corr[j]);
    q->h[j] += q->corr[j];                                       // h .+= correction :31
  }
  q->proj = sqrt(p);                                             // :28
  q->reorth = q->nrm < (1.0 / sqrt(2.0)) * q->proj;
}
// LinearAlgebra.givensAlgorithm(f, g) for complex arguments -> (c real, s, r) with [c s; -conj(s) c][f; g] = [r; 0]
// (c = |f| / d, s = (f / |f|) conj(g) / d, r = (f / |f|) d, d = hypot(|f|, |g|)).  For real f, g it differs from
// givens_real only in sign: (-c, -s, -r) when f < 0 and |f| <= |g| (and s = sign(g) when f == 0), which negates both
// rotated rows -- the back-substitution cancels it exactly.
B200_HD void givens_cplx(cplx<double> f, cplx<double> g, double &c, cplx<double> &s, cplx<double> &r) {
  if (g.re == 0.0 && g.im == 0.0) { c = 1.0; s = cplx<double>(0.0); r = f; return; }
  if (f.re == 0.0 && f.im == 0.0) {
    const double ag = hypot(g.re, g.im);
    c = 0.0; s = cplx<double>(g.re / ag, -g.im / ag); r = cplx<double>(ag); return;
  }
  const double f1 = hypot(f.re, f.im), g1 = hypot(g.re, g.im), d = hypot(f1, g1);
  const cplx<double> ph(f.re / f1, f.im / f1), t = ph * conj(g);
  c = f1 / d;
  s = cplx<double>(t.re / d, t.im / d);
  r = cplx<double>(ph.re * d, ph.im * d);
}
// ldiv!(FastHessenberg(H[1:m+1, 1:m]), rhs[1:m+1]) of src/hessenberg.jl:15-46, column-major H with leading dimension ldh
B200_HD void gm_hessenberg_solve_c(cplx<double> *H, int ldh, int m, cplx<double> *rhs) {
  for (int i = 0; i < m; ++i) {                                  // :24
    double c;
    cplx<double> s, r;
    givens_cplx(H[i + i * ldh], H[i + 1 + i * ldh], c, s, r);
    H[i + i * ldh] = c * H[i + i * ldh] + s * H[i + 1 + i * ldh];   // :28
    for (int j = i + 1; j < m; ++j) {                            // :31-35
      const cplx<double> a = H[i + j * ldh], b = H[i + 1 + j * ldh];
      H[i + j * ldh] = c * a + s * b;
      H[i + 1 + j * ldh] = -conj(s) * a + c * b;
    }
    const cplx<double> a = rhs[i], b = rhs[i + 1];               // :38-40
    rhs[i] = c * a + s * b;
    rhs[i + 1] = -conj(s) * a + c * b;
  }
  for (int i = m - 1; i >= 0; --i) {                             // UpperTriangular solve :44-45
    cplx<double> acc = rhs[i];
    for (int j = i + 1; j < m; ++j) acc -= H[i + j * ldh] * rhs[j];
    rhs[i] = acc / H[i + i * ldh];
  }
}
B200_HD void gm_step(GmScalC *q) {
  const int k = q->k, col = k - 1;
  cplx<double> *Hc = q->H + (size_t)col * kGmLdh;
  for (int j = 0; j < k; ++j) Hc[j] = q->h[j];                   // H[1:k, k] :68-73
  Hc[k] = cplx<double>(q->nrm);                                  // H[k+1, k] = orthogonalize_and_normalize!(...)
  if (q->nrm == 0.0) {                                           // update_residual! :224-233
    q->current = 0.0;
  } else {
    cplx<double> d(0.0);
    for (int j = 0; j < k; ++j) d += conj(q->nullvec[j]) * Hc[j];   // dot(nullvec[1:k], H[1:k, k])
    q->nullvec[k] = -conj(d / Hc[k]);                            // :229
    q->accumulator += abs2(q->nullvec[k]);                       // :230
    q->current = q->beta_res / sqrt(q->accumulator);
  }
  int flags = 0;
  const int k1 = k + 1;                                          // :78
  q->k = k1;
  if (k1 == q->restart + 1 || gm_done(q, q->iteration + 1)) {    // :82
    const int m = k1 - 1;                                        // solve_least_squares! :262-271
    for (int i = 0; i <= m; ++i) q->rhs[i] = cplx<double>(0.0);
    q->rhs[0] = cplx<double>(q->beta);                           // :265
    gm_hessenberg_solve_c(q->H, kGmLdh, m, q->rhs);
    q->m = m;
    q->k = 1;                                                    // :90
    flags |= GM_FIN;
    if (!gm_done(q, q->iteration)) flags |= GM_REINIT;           // :93 (sic: the old iteration count)
  }
  q->iteration += 1;
  if (q->hist && q->n_hist < q->hist_cap) q->hist[q->n_hist] = q->current;   // push!(history, :resnorm, ...) :211
  q->n_hist += 1;
  if (gm_done(q, q->iteration)) flags |= GM_DONE;                // :59
  if (!(q->current == q->current)) flags |= GM_DONE | GM_BREAKDOWN;
  q->flags = flags;
}

struct GmresOutcome {
  int64_t iters, mvps, n_hist;
  double residual, tol;
  int converged, breakdown, done, pad;
};

// ---- the driver in resumable pieces: scratch layout, setup (gmres_iterable! :108-136), advance (up to k calls of
// iterate :57-106), collect.  gmres_run is the one-shot form; the iterator of the C ABI keeps the scratch between calls.
template <typename T>
struct GmresLayout {
  T *V, *t1, *t2;
  int64_t ld;
  typename gm_scal<T>::type *s;
  double *hist;
  int64_t hist_cap;
};
inline size_t gm_vec_bytes(size_t elem, int64_t n) { return ((elem * (size_t)(n > 0 ? n : 1)) + 255) / 256 * 256; }
template <typename T>
size_t gmres_ws_bytes(int64_t n, int restart, int64_t hist_cap) {
  return gm_vec_bytes(sizeof(T), n) * (size_t)(restart + 3) + (sizeof(typename gm_scal<T>::type) + 255) / 256 * 256 +
         ((sizeof(double) * (size_t)(hist_cap > 0 ? hist_cap : 1)) + 255) / 256 * 256;
}
template <typename T>
GmresLayout<T> gmres_layout(void *ws, int64_t n, int restart, int64_t hist_cap) {
  const size_t vb = gm_vec_bytes(sizeof(T), n);
  GmresLayout<T> L;
  char *p = (char *)ws;
  L.V = (T *)p; p += vb * (size_t)(restart + 1);
  L.t1 = (T *)p; p += vb;
  L.t2 = (T *)p; p += vb;
  L.ld = (int64_t)(vb / sizeof(T));
  typedef typename gm_scal<T>::type Scal;
  L.s = (Scal *)p; p += (sizeof(Scal) + 255) / 256 * 256;
  L.hist = hist_cap > 0 ? (double *)p : nullptr;
  L.hist_cap = hist_cap > 0 ? hist_cap : 0;
  return L;
}

// The operators of one solve: A; Pl / Pr: preconditioner callbacks (y = P \ x) or nullptr; pl_diag / pr_diag: Jacobi
// diagonals or nullptr (Identity when both are null on a side).
template <typename T, typename B>
struct GmresOps {
  const typename B::Op *A, *Pl, *Pr;
  const T *pl_diag, *pr_diag;
};

// init! :235-255
template <typename T, typename B>
int gmres_init_residual(B &be, const GmresOps<T, B> &op, const GmresLayout<T> &L, int64_t n, const T *x, const T *b,
                        bool zero) {
  int s2;
  T *v0 = L.V, *t1 = L.t1, *t2 = L.t2;
  typename gm_scal<T>::type *s = L.s;
  if (!zero && (s2 = be.apply(op.A, x, t1))) return s2;                     // mul!(Ax, A, x) :245
  if (op.Pl) {
    if ((s2 = be.pass(GmResidual<T>{b, zero ? nullptr : t1, nullptr, t2, s, 0}, n))) return s2;
    if ((s2 = be.apply(op.Pl, t2, v0))) return s2;                          // ldiv!(Pl, first_col) :249
    if ((s2 = be.pass(GmNorm<T>{v0, s}, n))) return s2;
  } else {
    if ((s2 = be.pass(GmResidual<T>{b, zero ? nullptr : t1, op.pl_diag, v0, s, 1}, n))) return s2;
  }
  return be.pass(GmScale<T>{v0, &s->beta, (T)0}, n);                        // first_col .*= inv(beta) :253
}

template <typename T, typename B>
int gmres_setup(B &be, const GmresOps<T, B> &op, const GmresLayout<T> &L, int64_t n, int64_t n_global, T *x, const T *b,
                double abstol, double reltol, int restart, int64_t maxiter, int initially_zero, int64_t *mv_products) {
  if (reltol < 0) reltol = sqrt(eps_of<T>());                               // :187
  if (maxiter < 0) maxiter = n_global;                                      // :189
  if (restart < 1 || restart > kGmMaxRestart) return -1;                    // B200_ERR_INVALID (checked by the callers)
  int st;
  {
    typedef typename gm_scal<T>::type GmScal;
    std::unique_ptr<GmScal> h(new GmScal);
    memset(h.get(), 0, sizeof(GmScal));
    for (int i = 0; i < kGmLdh; ++i) h->nullvec[i] = 1.0;                   // ones(T, order + 1) :27
    h->accumulator = h->current = h->beta_res = h->beta = 1.0;
    h->abstol = abstol;
    h->reltol = reltol;
    h->maxiter = maxiter;
    h->hist = L.hist;
    h->hist_cap = L.hist_cap;
    h->k = 1;
    h->restart = restart;
    h->first = 1;
    if ((st = be.to_device(L.s, h.get(), sizeof(GmScal)))) return st;
  }
  if ((st = be.zero(L.V, gm_vec_bytes(sizeof(T), n) * (size_t)(restart + 1)))) return st;   // zeros(T, n, order + 1) :13
  *mv_products = initially_zero ? 1 : 0;                                    // :122 (sic)
  return gmres_init_residual<T, B>(be, op, L, n, x, b, initially_zero != 0);   // :126
}

// up to kmax more inner iterations (kmax < 0: until done); *mv_products is advanced by the products performed
template <typename T, typename B>
int gmres_advance(B &be, const GmresOps<T, B> &op, const GmresLayout<T> &L, int64_t n, T *x, const T *b, int orth_meth,
                  int64_t kmax, int64_t *mv_products) {
  T *V = L.V, *t1 = L.t1, *t2 = L.t2;
  const int64_t ld = L.ld;
  typedef typename gm_scal<T>::type GmScal;
  GmScal *s = L.s;
  const typename B::Op *A = op.A, *Pl = op.Pl, *Pr = op.Pr;
  const T *pl_diag = op.pl_diag, *pr_diag = op.pr_diag;
  auto col = [&](int j) { return V + (int64_t)j * ld; };
  const bool has_pr = Pr != nullptr || pr_diag != nullptr;
  int st;

  auto apply_prec = [&](const typename B::Op *P, const T *diag, const T *in, T *out) -> int {   // out = P \ in (out != in for callbacks)
    if (P) return be.apply(P, in, out);
    return be.pass(GmJacobi<T>{in, diag, out}, n);
  };
  auto expand = [&](int k) -> int {                                         // expand! :285-304, k 1-based
    int s2;
    T *next = col(k), *cur = col(k - 1);
    const T *src = cur;
    if (has_pr) {
      if ((s2 = apply_prec(Pr, pr_diag, cur, t1))) return s2;               // ldiv!(nextV, Pr, V[:, k]) :300
      src = t1;
    }
    if (Pl) {
      if ((s2 = be.apply(A, src, t2))) return s2;                           // mul! :287 / :293 / :301
      return be.apply(Pl, t2, next);                                        // ldiv!(Pl, nextV) :294 / :303
    }
    if ((s2 = be.apply(A, src, next))) return s2;
    if (pl_diag) return be.pass(GmJacobi<T>{next, pl_diag, next}, n);
    return 0;
  };
  auto orth = [&](int k) -> int {                                           // orthogonalize_and_normalize!(V[:, 1:k], V[:, k+1], H[1:k, k])
    int s2;
    T *w = col(k);
    if (orth_meth == GM_ORTH_MGS) {
      for (int i = 0; i <= k; ++i)
        if ((s2 = be.pass(GmMgs<T>{i > 0 ? col(i - 1) : nullptr, i < k ? col(i) : nullptr, w, s, i - 1, i, (T)0}, n)))
          return s2;
    } else {
      auto dots = [&](int to_corr) -> int {
        constexpr int DB = gm_dot_block<T>();
        for (int j0 = 0; j0 < k; j0 += DB) {
          const int cnt = k - j0 < DB ? k - j0 : DB;
          const int s3 = be.pass(GmDots<T>{col(j0), ld, cnt, j0, to_corr, w, s}, n);
          if (s3) return s3;
        }
        return 0;
      };
      auto update = [&](int which) -> int {
        for (int j0 = 0; j0 < k; j0 += kGmBlock) {
          const int cnt = k - j0 < kGmBlock ? k - j0 : kGmBlock;
          int s3;
          if (j0 + cnt == k) {
            GmUpdate<T, true> u{col(j0), ld, cnt, j0, which, -1.0, w, s, {}};
            s3 = be.pass(u, n);
          } else {
            GmUpdate<T, false> u{col(j0), ld, cnt, j0, which, -1.0, w, s, {}};
            s3 = be.pass(u, n);
          }
          if (s3) return s3;
        }
        return 0;
      };
      if ((s2 = dots(0))) return s2;                                        // mul!(h, V', w) :15 / :43
      if ((s2 = update(GM_COEF_H))) return s2;                              // mul!(w, V, h, -1, 1) ; nrm = norm(w) :16-17 / :44-45
      if (orth_meth == GM_ORTH_DGKS) {
        if ((s2 = be.scalar(ScalarStep<GmScal, gm_dgks_first>{s}))) return s2;
        for (;;) {                                                          // while nrm < eta * projection_size :26
          int again = 0;
          if ((s2 = be.read_flag(&s->reorth, &again))) return s2;
          if (!again) break;
          if ((s2 = dots(1))) return s2;                                    // correction = V' w :27
          if ((s2 = update(GM_COEF_CORR))) return s2;                       // mul!(w, V, correction, -1, 1) ; nrm :30, :32
          if ((s2 = be.scalar(ScalarStep<GmScal, gm_dgks_next>{s}))) return s2;   // :28, :31
        }
      }
    }
    return be.pass(GmScale<T>{w, &s->nrm, (T)0}, n);                        // w .*= inv(nrm) :36 / :48 / :76
  };
  auto update_solution = [&](int m) -> int {                                // update_solution! :273-283
    int s2;
    T *dst = x;
    if (has_pr) {
      if ((s2 = be.zero(t1, sizeof(T) * (size_t)n))) return s2;
      dst = t1;
    }
    for (int j0 = 0; j0 < m; j0 += kGmBlock) {
      const int cnt = m - j0 < kGmBlock ? m - j0 : kGmBlock;
      GmUpdate<T, false> u{col(j0), ld, cnt, j0, GM_COEF_Y, 1.0, dst, s, {}};
      if ((s2 = be.pass(u, n))) return s2;                                  // x += V[:, 1:k-1] y :275 / mul!(Ax, V, y) :280
    }
    if (has_pr) {
      if ((s2 = apply_prec(Pr, pr_diag, t1, t2))) return s2;                // ldiv!(Pr, Ax) :281
      if ((s2 = be.pass(GmAdd<T>{t2, x}, n))) return s2;                    // x .+= Ax :282
    }
    return 0;
  };

  int flags = 0, k = 1;
  if ((st = be.read_flag(&s->flags, &flags))) return st;
  if ((st = be.read_flag(&s->k, &k))) return st;                            // position inside the restart cycle
  int64_t performed = 0;
  while (!(flags & GM_DONE) && (kmax < 0 || performed < kmax)) {            // :59
    if ((st = expand(k))) return st;                                        // :63
    *mv_products += 1;                                                      // :65
    if ((st = orth(k))) return st;                                          // :68-73
    if ((st = be.scalar(ScalarStep<GmScal, gm_step>{s}))) return st;
    if ((st = be.read_flag(&s->flags, &flags))) return st;
    if (flags & GM_FIN) {
      if ((st = update_solution(k))) return st;                             // :85-88 (m = k columns)
      k = 1;
      if (flags & GM_REINIT) {
        if ((st = gmres_init_residual<T, B>(be, op, L, n, x, b, false))) return st;   // :96-99
        *mv_products += 1;                                                  // :101
      }
    } else {
      k += 1;
    }
    performed += 1;
    if (flags & GM_BREAKDOWN) break;
  }
  return 0;
}

template <typename T, typename B>
int gmres_collect(B &be, const GmresLayout<T> &L, int64_t mv_products, double *hist_host, GmresOutcome *out) {
  int st;
  typedef typename gm_scal<T>::type GmScal;
  std::unique_ptr<GmScal> h(new GmScal);
  if ((st = be.to_host(h.get(), L.s, sizeof(GmScal)))) return st;
  out->iters = h->iteration;
  out->mvps = mv_products;                                                  // history.mvps = iterable.mv_products :210
  out->residual = h->current;
  out->tol = h->tol;
  out->converged = h->current <= h->tol;                                    // :218
  out->breakdown = (h->flags & GM_BREAKDOWN) != 0;
  out->done = (h->flags & GM_DONE) != 0;
  out->n_hist = h->n_hist < L.hist_cap ? h->n_hist : L.hist_cap;
  if (hist_host && out->n_hist > 0 && (st = be.to_host(hist_host, L.hist, sizeof(double) * (size_t)out->n_hist))) return st;
  return 0;
}
template <typename B, typename Q>
int gmres_reset_window(B &be, Q *s) {
  const long long zero = 0;
  return be.to_device(&s->n_hist, &zero, sizeof(zero));
}

template <typename T, typename B>
int gmres_run(B &be, const typename B::Op *A, const typename B::Op *Pl, const typename B::Op *Pr, const T *pl_diag,
              const T *pr_diag, int64_t n, int64_t n_global, T *x, const T *b, double abstol, double reltol, int restart,
              int64_t maxiter, int initially_zero, int orth_meth, int64_t hist_cap, double *hist_host, GmresOutcome *out) {
  if (restart <= 0) restart = (int)(n_global < 20 ? n_global : 20);         // :188
  if (maxiter < 0) maxiter = n_global;                                      // :189
  if (restart > kGmMaxRestart) return -1;                                   // B200_ERR_INVALID (checked by the callers)
  if (!hist_host) hist_cap = 0;
  if (hist_cap > maxiter) hist_cap = maxiter;                               // reserve!(history, :resnorm, maxiter) :198
  void *ws = nullptr;
  int st = be.workspace(gmres_ws_bytes<T>(n, restart, hist_cap), &ws);
  if (st) return st;
  const GmresLayout<T> L = gmres_layout<T>(ws, n, restart, hist_cap);
  const GmresOps<T, B> op{A, Pl, Pr, pl_diag, pr_diag};
  int64_t mv_products = 0;
  if ((st = gmres_setup<T, B>(be, op, L, n, n_global, x, b, abstol, reltol, restart, maxiter, initially_zero, &mv_products)))
    return st;
  if ((st = gmres_advance<T, B>(be, op, L, n, x, b, orth_meth, -1, &mv_products))) return st;
  return gmres_collect<T, B>(be, L, mv_products, hist_host, out);
}

}  // namespace b200
