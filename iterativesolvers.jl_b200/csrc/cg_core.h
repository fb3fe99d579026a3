// cg_core.h -- cg!(x, A, b; Pl, ...) of reference src/cg.jl:209-242 (CGIterable iterate :43-66, PCGIterable iterate
// :72-100, cg_iterator! :120-155) written as fused passes (pass_core.h) for GENERAL operators and preconditioners:
// A (and Pl) may be device callbacks (`b200_linop`: the reference's duck-typed `mul!(y, A, x)` / `ldiv!(y, P, x)`
// contract, docs/src/getting_started.md:25-30, docs/src/preconditioning.md:5-15; test/cg.jl:71-77 runs cg on a
// LinearMap).  For a `b200_csr` operator with Identity / Jacobi the specialised engine of cg.cu (SpMV fused with its
// dot, three launches per iteration) is the fast path; this one keeps the same property that matters for a
// matrix-free operator: every scalar of the recurrence stays in device memory, the host never waits for a dot.
//
//   CG  (Pl = Identity)                                   PCG
//   C1  u = r + beta u                  :50-51            L   c = Pl \ r   (callback, or fused with D for Jacobi)  :79
//   S   c = A u                         :54               D   rho = <c, r> ; beta = rho / rho_prev                  :81-85
//   C2  alpha = residual^2 / <u, c>     :55               C1' u = c + beta u                                         :86
//   C3  x += alpha u ; r -= alpha c ; residual = ||r||    S, C2 (alpha = rho / <u, c>), C3                          :89-96
//                                       :58-62
// Algorithmic bytes per iteration besides the operator: CG 3 + 2 + 5 = 10 n V, PCG (Jacobi) 3 + 3 + 2 + 5 = 13 n V.
//
// Complex element types (T = cplx<R>): the scalar block is CgpScalC, where alpha, rho and beta are complex (fp64 for
// ComplexF32 too) and residual stays real; every dot is Julia's dot(x, y) = sum conj(x_i) y_i and takes two of a pass's
// sums (re, im).  The real instantiations are the code they were before complex types existed (if constexpr).
#pragma once
#include "complex.h"
#include "pass_core.h"

namespace b200 {

struct CgpScal {
  double residual, prev_residual, rho, tol, abstol, reltol;   // CGIterable / PCGIterable fields :5-30
  double alpha, beta;
  double sum[2];
  double *hist;
  long long hist_cap, n_hist;
  long long iteration, maxiter;                               // iteration starts at 0 (:34)
  int done, breakdown, precond, pad;
};

// complex element types: alpha, rho, beta complex (src/cg.jl:55, :82, :85), residual real
struct CgpScalC {
  double residual, prev_residual;
  cplx<double> rho;
  double tol, abstol, reltol;
  cplx<double> alpha, beta;
  double sum[2];
  double *hist;
  long long hist_cap, n_hist;
  long long iteration, maxiter;
  int done, breakdown, precond, pad;
};
template <typename T>
struct cgp_scal {
  typedef CgpScal type;
};
template <typename R>
struct cgp_scal<cplx<R>> {
  typedef CgpScalC type;
};

template <typename Q>
B200_HD void cgp_publish(Q *q, double residual) {             // after :62 / :96
  q->residual = residual;
  if (!(residual == residual)) q->breakdown = 1;
  if (q->hist && q->n_hist < q->hist_cap) q->hist[q->n_hist] = residual;
  q->n_hist += 1;
  q->iteration += 1;
  q->done = (q->iteration >= q->maxiter) || (q->residual <= q->tol) || q->breakdown;   // done() :36
}

// ---- cg_iterator! :126-141
template <typename T>
struct CgpInit {
  typedef typename cgp_scal<T>::type Scal;
  static constexpr int NRED = 1;
  const T *b, *ax;       // ax = A*x (nullptr when initially_zero)
  T *r, *u;
  Scal *s;
  B200_HD bool skip() const { return false; }
  B200_HD void load() {}
  B200_HD void elem(int64_t i, double *acc) const {
    T ri = b[i];                                       // copyto!(r, b) :130
    if (ax) ri = ri - ax[i];                           // r .-= c :138
    r[i] = ri;
    u[i] = (T)0;                                       // :129
    if constexpr (is_cplx<T>::value) acc[0] += (double)ri.re * (double)ri.re + (double)ri.im * (double)ri.im;
    else acc[0] += (double)ri * (double)ri;
  }
  B200_HD double *sums() const { return s->sum; }
  B200_HD void finish(const double *tot) const {
    Scal *q = s;
    q->residual = sqrt(tot[0]);                        // :140
    q->tol = fmax(q->reltol * q->residual, q->abstol); // :141
    q->prev_residual = 1.0;                            // one(residual) :146
    q->rho = 1.0;                                      // one(eltype(x)) :151
    q->beta = q->residual * q->residual;               // beta of the first CG step (:50 with prev_residual = 1)
    q->iteration = 0;
    q->n_hist = 0;
    q->breakdown = !(q->residual == q->residual);
    q->done = (q->iteration >= q->maxiter) || (q->residual <= q->tol) || q->breakdown;
  }
};

// ---- C1 / C1': u = z + beta u with z = r (CG) or z = c (PCG)
template <typename T>
struct CgpUpdateU {
  static constexpr int NRED = 0;
  const T *z;
  T *u;
  const typename cgp_scal<T>::type *s;
  T beta;
  B200_HD bool skip() const { return s->done != 0; }
  B200_HD void load() { beta = (T)s->beta; }
  B200_HD void elem(int64_t i, double *) const { u[i] = z[i] + beta * u[i]; }   // :51 / :86
  B200_HD double *sums() const { return nullptr; }
  B200_HD void finish(const double *) const {}
};

// ---- D: rho = <c, r> (PCG).  With a Jacobi preconditioner the pass also forms c = r ./ d.
template <typename T>
struct CgpRho {
  static constexpr int NRED = is_cplx<T>::value ? 2 : 1;
  T *c;
  const T *r, *diag;     // diag: Jacobi (c is written here); nullptr: c was produced by the preconditioner callback
  typename cgp_scal<T>::type *s;
  B200_HD bool skip() const { return s->done != 0; }
  B200_HD void load() {}
  B200_HD void elem(int64_t i, double *acc) const {
    const T ri = r[i];
    T ci;
    if (diag) {
      ci = ri / diag[i];                               // ldiv!(c, Pl, r) :79
      c[i] = ci;
    } else {
      ci = c[i];
    }
    if constexpr (is_cplx<T>::value) {                 // dot(c, r) = sum conj(c_i) r_i :82
      acc[0] += (double)ci.re * (double)ri.re + (double)ci.im * (double)ri.im;
      acc[1] += (double)ci.re * (double)ri.im - (double)ci.im * (double)ri.re;
    } else {
      acc[0] += (double)ci * (double)ri;               // dot(c, r) :82
    }
  }
  B200_HD double *sums() const { return s->sum; }
  B200_HD void finish(const double *tot) const {
    if constexpr (is_cplx<T>::value) {
      const cplx<double> rho_prev = s->rho;            // :81
      s->rho = cplx<double>(tot[0], tot[1]);           // :82
      s->beta = s->rho / rho_prev;                     // :85
    } else {
      const double rho_prev = s->rho;                  // :81
      s->rho = tot[0];                                 // :82
      s->beta = s->rho / rho_prev;                     // :85
    }
  }
};

// ---- C2: alpha
template <typename T>
struct CgpAlpha {
  static constexpr int NRED = is_cplx<T>::value ? 2 : 1;
  const T *u, *c;
  typename cgp_scal<T>::type *s;
  B200_HD bool skip() const { return s->done != 0; }
  B200_HD void load() {}
  B200_HD void elem(int64_t i, double *acc) const {
    if constexpr (is_cplx<T>::value) {                 // dot(u, c) = sum conj(u_i) c_i
      const T ui = u[i], ci = c[i];
      acc[0] += (double)ui.re * (double)ci.re + (double)ui.im * (double)ci.im;
      acc[1] += (double)ui.re * (double)ci.im - (double)ui.im * (double)ci.re;
    } else {
      acc[0] += (double)u[i] * (double)c[i];
    }
  }
  B200_HD double *sums() const { return s->sum; }
  B200_HD void finish(const double *tot) const {
    if constexpr (is_cplx<T>::value)
      s->alpha = (s->precond ? s->rho : cplx<double>(s->residual * s->residual)) / cplx<double>(tot[0], tot[1]);
    else
      s->alpha = (s->precond ? s->rho : s->residual * s->residual) / tot[0];   // :90 / :55
  }
};

// ---- C3
template <typename T>
struct CgpUpdateXR {
  typedef typename cgp_scal<T>::type Scal;
  static constexpr int NRED = 1;
  T *x, *r;
  const T *u, *c;
  Scal *s;
  T alpha;
  B200_HD bool skip() const { return s->done != 0; }
  B200_HD void load() { alpha = (T)s->alpha; }
  B200_HD void elem(int64_t i, double *acc) const {
    x[i] = x[i] + alpha * u[i];                        // :58 / :93
    const T ri = r[i] - alpha * c[i];                  // :59 / :94
    r[i] = ri;
    if constexpr (is_cplx<T>::value) acc[0] += (double)ri.re * (double)ri.re + (double)ri.im * (double)ri.im;
    else acc[0] += (double)ri * (double)ri;
  }
  B200_HD double *sums() const { return s->sum; }
  B200_HD void finish(const double *tot) const {
    Scal *q = s;
    const double res = sqrt(tot[0]);                   // :62 / :96
    if (!q->precond) {
      q->prev_residual = q->residual;                  // :61
      q->beta = (res * res) / (q->prev_residual * q->prev_residual);   // :50 of the next step
    }
    cgp_publish(q, res);
  }
};

struct CgpOutcome {
  int64_t iters, mvps, n_hist;
  double residual, tol;
  int converged, breakdown, done, pad;
};

// ---- the driver in resumable pieces (cg_iterator! :120-155 = setup, iterate :43-100 = advance); cgp_run is the one-shot
// form, the iterator of the C ABI keeps the scratch between calls.
template <typename T>
struct CgpLayout {
  T *u, *r, *c;
  typename cgp_scal<T>::type *s;
  double *hist;
  int64_t hist_cap;
};
inline size_t cgp_vec_bytes(size_t elem, int64_t n) { return ((elem * (size_t)(n > 0 ? n : 1)) + 255) / 256 * 256; }
template <typename T>
size_t cgp_ws_bytes(int64_t n, int64_t hist_cap) {
  return 3 * cgp_vec_bytes(sizeof(T), n) + 512 + ((sizeof(double) * (size_t)(hist_cap > 0 ? hist_cap : 1)) + 255) / 256 * 256;
}
template <typename T>
CgpLayout<T> cgp_layout(void *ws, int64_t n, int64_t hist_cap) {
  static_assert(sizeof(CgpScal) <= 512 && sizeof(CgpScalC) <= 512, "CgpScal outgrew its slot");
  const size_t vb = cgp_vec_bytes(sizeof(T), n);
  CgpLayout<T> L;
  char *p = (char *)ws;
  L.u = (T *)p; p += vb;
  L.r = (T *)p; p += vb;
  L.c = (T *)p; p += vb;
  L.s = (typename cgp_scal<T>::type *)p; p += 512;
  L.hist = hist_cap > 0 ? (double *)p : nullptr;
  L.hist_cap = hist_cap > 0 ? hist_cap : 0;
  return L;
}

// A: the operator; Pl: preconditioner callback (y = Pl \ x) or nullptr; diag: Jacobi diagonal or nullptr (Identity
// when both are null).  x, b: n values.
template <typename T, typename B>
int cgp_setup(B &be, const typename B::Op *A, bool precond, const CgpLayout<T> &L, int64_t n, int64_t n_global, T *x,
              const T *b, double abstol, double reltol, int64_t maxiter, int initially_zero, int64_t *mvps0) {
  if (reltol < 0) reltol = sqrt(eps_of<T>());                               // :211
  if (maxiter < 0) maxiter = n_global;                                      // :212
  typename cgp_scal<T>::type h;
  memset(&h, 0, sizeof(h));
  h.abstol = abstol;
  h.reltol = reltol;
  h.maxiter = maxiter;
  h.hist = L.hist;
  h.hist_cap = L.hist_cap;
  h.precond = precond;
  int st;
  if ((st = be.to_device(L.s, &h, sizeof(h)))) return st;
  *mvps0 = 0;
  if (!initially_zero) {                                                    // :133-139
    if ((st = be.apply(A, x, L.c))) return st;
    *mvps0 = 1;
  }
  return be.pass(CgpInit<T>{b, initially_zero ? nullptr : L.c, L.r, L.u, L.s}, n);
}

// up to k more iterations (k < 0: until done)
template <typename T, typename B>
int cgp_advance(B &be, const typename B::Op *A, const typename B::Op *Pl, const T *diag, const CgpLayout<T> &L, int64_t n,
                T *x, int64_t k, int check_every) {
  int st;
  T *u = L.u, *r = L.r, *c = L.c;
  typename cgp_scal<T>::type *s = L.s;
  typename cgp_scal<T>::type h;
  if ((st = be.to_host(&h, s, sizeof(h)))) return st;
  if (h.done) return 0;
  const bool precond = Pl != nullptr || diag != nullptr;
  const int64_t left = h.maxiter - h.iteration;
  const int64_t todo = (k < 0 || k > left) ? left : k;
  if (check_every <= 0) check_every = 16;
  int64_t enqueued = 0;
  for (;;) {
    int done = 0;
    if ((st = be.read_flag(&s->done, &done))) return st;
    if (done || enqueued >= todo) break;
    const int64_t batch = check_every < todo - enqueued ? check_every : todo - enqueued;
    for (int64_t q = 0; q < batch; ++q) {
      if (precond) {
        if (Pl && (st = be.apply(Pl, r, c))) return st;                                        // L  :79
        if ((st = be.pass(CgpRho<T>{c, r, Pl ? nullptr : diag, s}, n))) return st;              // D  :81-85
        if ((st = be.pass(CgpUpdateU<T>{c, u, s}, n))) return st;                               // C1' :86
      } else {
        if ((st = be.pass(CgpUpdateU<T>{r, u, s}, n))) return st;                               // C1 :51
      }
      if ((st = be.apply(A, u, c))) return st;                                                 // S  :54 / :89
      if ((st = be.pass(CgpAlpha<T>{u, c, s}, n))) return st;                                   // C2
      if ((st = be.pass(CgpUpdateXR<T>{x, r, u, c, s}, n))) return st;                          // C3
    }
    enqueued += batch;
  }
  return 0;
}

template <typename T, typename B>
int cgp_collect(B &be, const CgpLayout<T> &L, int64_t mvps0, double *hist_host, CgpOutcome *out) {
  int st;
  typename cgp_scal<T>::type h;
  if ((st = be.to_host(&h, L.s, sizeof(h)))) return st;
  out->iters = h.iteration;
  out->mvps = mvps0 + h.iteration;
  out->residual = h.residual;
  out->tol = h.tol;
  out->converged = h.residual <= h.tol;                                     // converged() :32
  out->breakdown = h.breakdown;
  out->done = h.done;
  out->n_hist = h.n_hist < L.hist_cap ? h.n_hist : L.hist_cap;
  if (hist_host && out->n_hist > 0 && (st = be.to_host(hist_host, L.hist, sizeof(double) * (size_t)out->n_hist))) return st;
  return 0;
}
template <typename B, typename Q>
int cgp_reset_window(B &be, Q *s) {
  const long long zero = 0;
  return be.to_device(&s->n_hist, &zero, sizeof(zero));
}

template <typename T, typename B>
int cgp_run(B &be, const typename B::Op *A, const typename B::Op *Pl, const T *diag, int64_t n, int64_t n_global, T *x,
            const T *b, double abstol, double reltol, int64_t maxiter, int initially_zero, int check_every,
            int64_t hist_cap, double *hist_host, CgpOutcome *out) {
  if (maxiter < 0) maxiter = n_global;
  if (!hist_host) hist_cap = 0;
  if (hist_cap > maxiter + 1) hist_cap = maxiter + 1;
  void *ws = nullptr;
  int st = be.workspace(cgp_ws_bytes<T>(n, hist_cap), &ws);
  if (st) return st;
  const CgpLayout<T> L = cgp_layout<T>(ws, n, hist_cap);
  int64_t mvps0 = 0;
  if ((st = cgp_setup<T, B>(be, A, Pl != nullptr || diag != nullptr, L, n, n_global, x, b, abstol, reltol, maxiter,
                            initially_zero, &mvps0)))
    return st;
  if ((st = cgp_advance<T, B>(be, A, Pl, diag, L, n, x, -1, check_every))) return st;
  return cgp_collect<T, B>(be, L, mvps0, hist_host, out);
}

}  // namespace b200
